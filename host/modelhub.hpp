// host/modelhub.hpp — C++ mirror of the Go API the north_star adds to kukeon (the reference is compiled Go and
// Go is not installed here, so the host side above the C ABI is written in C++):
//
//   kukeon::gpupool::Pool / Model   <->  internal/gpupool (cgo wrapper, INTEGRATION.md §1)
//   kukeon::modelhub::Pull/Load/Mount <-> internal/modelhub additions (INTEGRATION.md §2)
//   kukeon::errdefs::*              <->  sentinel errors, internal/errdefs/errdefs.go:23-
//
// Header-only; every call goes through include/kukeon_gpuload.h.  No tensor byte is touched on the host.
#pragma once
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../include/kukeon_gpuload.h"

namespace kukeon {

namespace errdefs {
// One class per sentinel the Go shim would add; `code` keeps the kk_status for callers that switch on it.
struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(std::string(kk_status_name(c)) + ": " + m), code(c) {}
};
struct ErrGPUPoolModelNotFound : Error { using Error::Error; };
struct ErrGPUPoolBadCheckpoint : Error { using Error::Error; };
struct ErrGPUPoolNoMemory : Error { using Error::Error; };
struct ErrGPUPoolBusy : Error { using Error::Error; };
struct ErrGPUPoolUnsupported : Error { using Error::Error; };
struct ErrGPUPoolLoad : Error { using Error::Error; };

inline void check(int rc) {
  if (rc == KK_OK) return;
  const std::string msg = kk_last_error();
  switch (rc) {
    case KK_ENOENT: throw ErrGPUPoolModelNotFound(rc, msg);
    case KK_EFORMAT: throw ErrGPUPoolBadCheckpoint(rc, msg);
    case KK_ENOMEM: throw ErrGPUPoolNoMemory(rc, msg);
    case KK_EBUSY: throw ErrGPUPoolBusy(rc, msg);
    case KK_EUNSUPPORTED: throw ErrGPUPoolUnsupported(rc, msg);
    default: throw ErrGPUPoolLoad(rc, msg);
  }
}
}  // namespace errdefs

namespace gpupool {

// Load flags (kk_load_opts.flags), the names the Go package gives them; the models[].options of a manifest map onto these.
constexpr uint32_t kFlagGPT2Conv1DTranspose = KK_LOAD_GPT2_CONV1D_T;
constexpr uint32_t kFlagKeepF32 = KK_LOAD_KEEP_F32;
constexpr uint32_t kFlagF8ToBF16 = KK_LOAD_F8_TO_BF16;
constexpr uint32_t kFlagF16 = KK_LOAD_F16;  // every float output as IEEE fp16 instead of bf16, same pool layout
constexpr uint32_t kFlagHFLayout = KK_LOAD_HF_LAYOUT;  // GGUF in Hugging Face layout: HF names, one tensor per expert, Q/K rows un-permuted

struct Config {
  std::vector<int> devices{0};
  uint64_t pool_bytes_per_device = 0;
  uint32_t staging_buffers = 0;
  uint64_t staging_buffer_bytes = 0;
  uint32_t reader_threads = 0;
  uint32_t flags = 0;
};

class Model {
 public:
  Model() = default;
  explicit Model(kk_model* h) : h_(h) {}
  Model(Model&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  Model& operator=(Model&& o) noexcept {
    if (this != &o) { reset(); h_ = o.h_; o.h_ = nullptr; }
    return *this;
  }
  Model(const Model&) = delete;
  Model& operator=(const Model&) = delete;
  ~Model() { reset(); }

  void Acquire() { errdefs::check(kk_acquire(h_)); }
  // Drops the reference this object holds (idempotent).
  void Release() { reset(); }
  // Extra references taken with Acquire() are dropped with this one.
  void ReleaseOne() { errdefs::check(kk_release(h_)); }

  kk_model_info Info() const {
    kk_model_info mi;
    errdefs::check(kk_model_get_info(h_, &mi));
    return mi;
  }
  std::vector<kk_placement> Placements(const std::string& tensor) const {
    kk_placement out[KK_MAX_DEVICES];
    size_t n = 0;
    errdefs::check(kk_placements(h_, tensor.c_str(), out, KK_MAX_DEVICES, &n));
    return std::vector<kk_placement>(out, out + n);
  }
  // (64-byte IPC handle, manifest JSON) of `device`'s pool.
  std::pair<std::string, std::string> Export(int device) const {
    size_t need = 0;
    errdefs::check(kk_export_size(h_, device, &need));
    std::string man(need, '\0'), handle(KK_IPC_HANDLE_BYTES, '\0');
    errdefs::check(kk_export(h_, device, &handle[0], &man[0], need));
    man.resize(need - 1);
    return {handle, man};
  }
  std::string Manifest(int device) const {
    size_t need = 0;
    errdefs::check(kk_export_size(h_, device, &need));
    std::string man(need, '\0');
    errdefs::check(kk_export(h_, device, nullptr, &man[0], need));
    man.resize(need - 1);
    return man;
  }
  std::string Stats() const {
    std::string s(1 << 16, '\0');
    errdefs::check(kk_stats(h_, &s[0], s.size()));
    s.resize(strlen(s.c_str()));
    return s;
  }
  uint64_t Checksum(int device, uint64_t off, uint64_t n) const {
    uint64_t v = 0;
    errdefs::check(kk_checksum(h_, device, off, n, &v));
    return v;
  }
  kk_model* handle() const { return h_; }
  // kk_derive_adapter: the model Pool::Load(<this model's path and options>, adapter) returns, built from this model's resident pools on the
  // GPU.  A model of its own; this one may be released at once.
  Model Derive(const std::string& adapter) const {
    kk_model* m = nullptr;
    errdefs::check(kk_derive_adapter(h_, adapter.c_str(), &m));
    return Model(m);
  }

 private:
  void reset() {
    if (h_) { kk_release(h_); h_ = nullptr; }
  }
  kk_model* h_ = nullptr;
};

// Pipeline stage: layers [begin, end) of a checkpoint (kk_load_opts.layer_begin / layer_end); {0, 0} is the whole checkpoint.
struct Layers {
  uint32_t begin = 0, end = 0;
};

class Pool {
 public:
  explicit Pool(const Config& cfg) {
    kk_config c{};
    c.n_devices = (int32_t)cfg.devices.size();
    for (size_t i = 0; i < cfg.devices.size() && i < KK_MAX_DEVICES; ++i) c.devices[i] = cfg.devices[i];
    c.pool_bytes_per_device = cfg.pool_bytes_per_device;
    c.n_staging_buffers = cfg.staging_buffers;
    c.staging_buffer_bytes = cfg.staging_buffer_bytes;
    c.n_reader_threads = cfg.reader_threads;
    c.flags = cfg.flags;
    errdefs::check(kk_open(&c, &h_));
  }
  Pool(const Pool&) = delete;
  Pool& operator=(const Pool&) = delete;
  ~Pool() {
    if (h_) kk_close(h_);
  }
  void Close() {
    if (h_) { errdefs::check(kk_close(h_)); h_ = nullptr; }
  }
  // layers: the pipeline stage [begin, end) to load; {0, 0} is the whole checkpoint.  A stage is a model of its own.
  // adapter: a PEFT LoRA adapter merged into the pool(s) after the load (kk_load_adapter); empty: the checkpoint alone.  Base + adapter is a
  // model of its own.
  Model Load(const std::string& path, int mode = KK_MODE_SINGLE, int fanout = KK_FANOUT_P2P, uint32_t flags = 0, Layers layers = {},
             const std::string& adapter = std::string()) {
    kk_load_opts o{};
    o.mode = mode;
    o.fanout = fanout;
    o.flags = flags;
    o.layer_begin = layers.begin;
    o.layer_end = layers.end;
    kk_model* m = nullptr;
    if (adapter.empty()) errdefs::check(kk_load_ex(h_, path.c_str(), &o, &m));
    else errdefs::check(kk_load_adapter(h_, path.c_str(), &o, adapter.c_str(), &m));
    return Model(m);
  }
  kk_ctx* handle() const { return h_; }

 private:
  kk_ctx* h_ = nullptr;
};

}  // namespace gpupool

namespace modelhub {

struct TensorIndex {
  std::vector<std::string> shards;
  std::vector<kk_tensor_meta> tensors;
  uint64_t file_bytes() const {
    uint64_t n = 0;
    for (auto& t : tensors) n += t.nbytes;
    return n;
  }
};

// Pull: resolve a local checkpoint path and index it (CPU only).
inline TensorIndex Pull(const std::string& path) {
  TensorIndex ix;
  kk_tensor_meta* recs = nullptr;
  size_t n = 0;
  errdefs::check(kk_index(nullptr, path.c_str(), &recs, &n));
  ix.tensors.assign(recs, recs + n);
  kk_free_index(recs);
  size_t ns = 0;
  errdefs::check(kk_index_shard(nullptr, path.c_str(), 0, nullptr, 0, &ns));
  char buf[4096];
  for (size_t i = 0; i < ns; ++i) {
    errdefs::check(kk_index_shard(nullptr, path.c_str(), i, buf, sizeof buf, nullptr));
    ix.shards.emplace_back(buf);
  }
  return ix;
}

inline gpupool::Model Load(gpupool::Pool& pool, const std::string& path, int mode = KK_MODE_SINGLE, uint32_t flags = 0,
                           gpupool::Layers layers = {}, const std::string& adapter = std::string()) {
  return pool.Load(path, mode, KK_FANOUT_P2P, flags, layers, adapter);
}

// Derive: base + a PEFT LoRA adapter built from the resident base on the GPU, the model Load(pool, base's path, ..., adapter) returns.
inline gpupool::Model Derive(const gpupool::Model& base, const std::string& adapter) { return base.Derive(adapter); }

struct OCIMount { std::string destination, type, source; std::vector<std::string> options; };
struct MountSpec {
  std::vector<OCIMount> mounts;
  std::vector<std::string> env;
  std::string host_dir;
};

namespace detail {
// tmp + fsync + rename, the pattern of internal/metadata/metadata.go:105-140.
inline void atomic_write(const std::string& file, const std::string& data, mode_t mode) {
  std::string tmp = file + ".tmpXXXXXX";
  int fd = mkstemp(&tmp[0]);
  if (fd < 0) throw errdefs::ErrGPUPoolLoad(KK_EIO, "mkstemp " + tmp + ": " + strerror(errno));
  bool ok = fchmod(fd, mode) == 0 && write(fd, data.data(), data.size()) == (ssize_t)data.size() && fsync(fd) == 0;
  close(fd);
  if (!ok || rename(tmp.c_str(), file.c_str()) != 0) {
    unlink(tmp.c_str());
    throw errdefs::ErrGPUPoolLoad(KK_EIO, "write " + file + ": " + strerror(errno));
  }
}
inline void mkdir_p(const std::string& d) {
  for (size_t i = 1; i <= d.size(); ++i)
    if (i == d.size() || d[i] == '/') {
      std::string p = d.substr(0, i);
      if (mkdir(p.c_str(), 0750) != 0 && errno != EEXIST) throw errdefs::ErrGPUPoolLoad(KK_EIO, "mkdir " + p + ": " + strerror(errno));
    }
}
}  // namespace detail

// Mount: stage <container_dir>/gpupool/{manifest.json,ipc.handle} and describe the read-only bind mount + env a
// ctr.WithGPUWeights BuildOption (INTEGRATION.md §3) adds to the container's OCI spec.
inline MountSpec Mount(const gpupool::Model& m, int device, const std::string& container_dir) {
  auto ex = m.Export(device);
  MountSpec s;
  s.host_dir = container_dir + "/gpupool";
  detail::mkdir_p(s.host_dir);
  detail::atomic_write(s.host_dir + "/manifest.json", ex.second, 0644);
  detail::atomic_write(s.host_dir + "/ipc.handle", ex.first, 0640);
  s.mounts.push_back({"/run/kukeon/gpupool", "bind", s.host_dir, {"rbind", "ro"}});
  // the GPU is named by UUID / PCI bus id (kk_device_identity): the daemon's CUDA ordinal means nothing inside the container
  char bus[32] = "", uuid[64] = "";
  if (kk_device_identity(device, bus, sizeof bus, uuid, sizeof uuid) != KK_OK) throw errdefs::ErrGPUPoolLoad(KK_ECUDA, std::string("kk_device_identity: ") + kk_last_error());
  s.env = {"KUKEON_GPUPOOL_MANIFEST=/run/kukeon/gpupool/manifest.json", "KUKEON_GPUPOOL_IPC_HANDLE=/run/kukeon/gpupool/ipc.handle",
           std::string("KUKEON_GPUPOOL_DEVICE_UUID=") + uuid, std::string("KUKEON_GPUPOOL_PCI_BUS_ID=") + bus};
  return s;
}

}  // namespace modelhub
}  // namespace kukeon
