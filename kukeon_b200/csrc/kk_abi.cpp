// extern "C" surface of libkukeon_gpuload.so (see include/kukeon_gpuload.h for the contract and the
// reference seams each entry point would be bound next to).  Every function catches everything and
// maps it to a negative kk_status + thread-local message — nothing C++ crosses the boundary.
#include <cstring>
#include <new>

#include "kk_loader.hpp"

namespace kk {
static thread_local std::string g_last_error;
void set_last_error(const std::string& s) { g_last_error = s; }
const char* get_last_error() { return g_last_error.c_str(); }
}  // namespace kk

namespace {

template <class F>
int guard(F&& f) {
  try {
    f();
    return KK_OK;
  } catch (const kk::Error& e) {
    kk::set_last_error(e.what());
    return e.code;
  } catch (const std::bad_alloc&) {
    kk::set_last_error("out of host memory");
    return KK_ENOMEM;
  } catch (const std::exception& e) {
    kk::set_last_error(std::string("internal error: ") + e.what());
    return KK_ESTATE;
  } catch (...) {
    kk::set_last_error("internal error: unknown exception");
    return KK_ESTATE;
  }
}

void need(const void* p, const char* what) {
  if (!p) kk::fail(KK_EINVAL, "%s is NULL", what);
}

void fill_meta(const kk::TensorRec& t, kk_tensor_meta* o) {
  memset(o, 0, sizeof *o);
  strncpy(o->name, t.name.c_str(), KK_NAME_MAX - 1);
  o->dtype = t.dtype;
  o->n_dims = (uint32_t)t.shape.size();
  for (size_t d = 0; d < t.shape.size(); ++d) o->shape[d] = t.shape[d];
  o->shard = t.shard;
  o->file_offset = t.file_offset;
  o->nbytes = t.nbytes;
}

}  // namespace

#pragma GCC visibility push(default)
extern "C" {

int kk_abi_version(void) { return KK_ABI_VERSION; }

const char* kk_last_error(void) { return kk::get_last_error(); }

const char* kk_status_name(int s) {
  switch (s) {
    case KK_OK: return "KK_OK";
    case KK_EINVAL: return "KK_EINVAL";
    case KK_ENOENT: return "KK_ENOENT";
    case KK_EFORMAT: return "KK_EFORMAT";
    case KK_EIO: return "KK_EIO";
    case KK_ENOMEM: return "KK_ENOMEM";
    case KK_ECUDA: return "KK_ECUDA";
    case KK_EUNSUPPORTED: return "KK_EUNSUPPORTED";
    case KK_EBUSY: return "KK_EBUSY";
    case KK_ERANGE: return "KK_ERANGE";
    case KK_ESTATE: return "KK_ESTATE";
    default: return "KK_?";
  }
}

int kk_open(const kk_config* cfg, kk_ctx** out) {
  return guard([&] {
    need(cfg, "cfg");
    need(out, "out");
    *out = nullptr;
    *out = kk::ctx_open(*cfg);
  });
}

int kk_close(kk_ctx* ctx) {
  return guard([&] {
    need(ctx, "ctx");
    kk::ctx_close(ctx);
  });
}

int kk_index(kk_ctx*, const char* path, kk_tensor_meta** out, size_t* n) {
  return guard([&] {
    need(path, "path");
    need(out, "out");
    need(n, "n");
    *out = nullptr;
    *n = 0;
    kk::Index ix = kk::index_path(path);
    kk_tensor_meta* recs = (kk_tensor_meta*)calloc(ix.tensors.size() ? ix.tensors.size() : 1, sizeof(kk_tensor_meta));
    if (!recs) kk::fail(KK_ENOMEM, "out of host memory for %zu index records", ix.tensors.size());
    for (size_t i = 0; i < ix.tensors.size(); ++i) fill_meta(ix.tensors[i], &recs[i]);
    *out = recs;
    *n = ix.tensors.size();
  });
}

int kk_free_index(kk_tensor_meta* recs) {
  free(recs);
  return KK_OK;
}

int kk_index_shard(kk_ctx*, const char* path, size_t i, char* buf, size_t cap, size_t* n_out) {
  return guard([&] {
    need(path, "path");
    kk::Index ix = kk::index_path(path);
    if (n_out) *n_out = ix.shards.size();
    if (!buf) return;
    if (i >= ix.shards.size()) kk::fail(KK_EINVAL, "shard %zu out of range (%zu shards)", i, ix.shards.size());
    if (ix.shards[i].size() + 1 > cap) kk::fail(KK_ERANGE, "need %zu bytes", ix.shards[i].size() + 1);
    memcpy(buf, ix.shards[i].c_str(), ix.shards[i].size() + 1);
  });
}

int kk_plan_describe(kk_ctx*, const char* path, const kk_load_opts* opts, int n_parts, uint64_t chunk_bytes, char* json,
                     size_t cap, size_t* required) {
  return guard([&] {
    need(path, "path");
    need(opts, "opts");
    if (chunk_bytes == 0) chunk_bytes = 64ull << 20;
    kk::Plan P = kk::build_plan(kk::index_path(path), opts->mode, opts->flags & ~KK_LOAD_DEFER, n_parts, chunk_bytes);
    std::string s = kk::plan_to_json(P);
    if (required) *required = s.size() + 1;
    if (!json) return;
    if (s.size() + 1 > cap) kk::fail(KK_ERANGE, "plan description needs %zu bytes", s.size() + 1);
    memcpy(json, s.c_str(), s.size() + 1);
  });
}

int kk_load(kk_ctx* ctx, const char* path, int mode, int fanout, kk_model** out) {
  kk_load_opts o{};
  o.mode = mode;
  o.fanout = fanout;
  return kk_load_ex(ctx, path, &o, out);
}

int kk_load_ex(kk_ctx* ctx, const char* path, const kk_load_opts* opts, kk_model** out) {
  return guard([&] {
    need(ctx, "ctx");
    need(path, "path");
    need(opts, "opts");
    need(out, "out");
    *out = nullptr;
    *out = kk::model_load(ctx, path, *opts);
  });
}

int kk_load_part(kk_model* m) {
  return guard([&] {
    need(m, "model");
    kk::model_load_part(m);
  });
}

int kk_peer_attach(kk_model* m, int rank, const void* h) {
  return guard([&] {
    need(m, "model");
    need(h, "ipc_handle");
    kk::model_peer_attach(m, kk::kPeerPool, rank, h, true);
  });
}

int kk_peer_detach_all(kk_model* m) {
  return guard([&] {
    need(m, "model");
    kk::model_peer_detach_all(m);
  });
}

// KK_BUF_* -> the peer buffer it names and whether its handle is a device pointer rather than a CUDA IPC handle; false for an unknown kind.
static bool buf_kind(int which, kk::PeerKind& kind, bool& by_ptr) {
  by_ptr = which == KK_BUF_POOL_PTR || which == KK_BUF_SLICE_PTR;
  switch (which) {
    case KK_BUF_POOL: case KK_BUF_POOL_PTR: kind = kk::kPeerPool; return true;
    case KK_BUF_RAW: kind = kk::kPeerRaw; return true;
    case KK_BUF_SLICE: case KK_BUF_SLICE_PTR: kind = kk::kPeerSlice; return true;
  }
  return false;
}

int kk_export_buffer(kk_model* m, int device, int which, void* h) {
  return guard([&] {
    need(m, "model");
    need(h, "ipc_handle");
    int li = kk::model_local_device(m, device);
    kk::PeerKind kind;
    bool by_ptr;
    if (!buf_kind(which, kind, by_ptr) || (kind == kk::kPeerPool && by_ptr)) kk::fail(KK_EINVAL, "unknown buffer kind %d", which);
    if (kind == kk::kPeerPool) {
      if (m->pools[(size_t)li].is_nvls()) kk::fail(KK_EUNSUPPORTED, "pools of a KK_FANOUT_NVLS model cannot be exported over CUDA IPC");
      kk::model_pool_ipc_handle(m, li, h);
    } else if (kind == kk::kPeerRaw) {
      kk::model_export_raw(m, li, h);
    } else {
      kk::model_export_slice(m, h, by_ptr);
    }
  });
}

int kk_peer_attach_buffer(kk_model* m, int rank, int which, const void* h) {
  return guard([&] {
    need(m, "model");
    need(h, "ipc_handle");
    kk::PeerKind kind;
    bool by_ptr;
    if (!buf_kind(which, kind, by_ptr)) kk::fail(KK_EINVAL, "unknown buffer kind %d", which);
    kk::model_peer_attach(m, kind, rank, h, !by_ptr);
  });
}

int kk_convert_local(kk_model* m, float* ms_total) {
  return guard([&] {
    need(m, "model");
    kk::model_convert_local(m, ms_total);
  });
}

int kk_model_get_info(kk_model* m, kk_model_info* o) {
  return guard([&] {
    need(m, "model");
    need(o, "out");
    memset(o, 0, sizeof *o);
    o->n_tensors = m->plan.index.tensors.size();
    o->n_shards = m->plan.index.shards.size();
    o->file_bytes = m->plan.file_bytes;
    uint64_t pb = 0;
    for (auto& pool : m->pools) pb = pool.bytes > pb ? pool.bytes : pb;
    o->pool_bytes = pb;
    o->n_devices = (int32_t)m->dev_idx.size();
    for (size_t i = 0; i < m->dev_idx.size(); ++i) o->devices[i] = m->ctx->devs[(size_t)m->dev_idx[i]].ordinal;
    o->mode = m->plan.mode;
    {
      std::lock_guard<std::mutex> g(m->ctx->mu);
      o->refcount = m->refcount;
      o->loaded = m->loaded ? 1 : 0;
    }
  });
}

int kk_model_tensor(kk_model* m, size_t i, kk_tensor_meta* out) {
  return guard([&] {
    need(m, "model");
    need(out, "out");
    if (i >= m->plan.index.tensors.size()) kk::fail(KK_EINVAL, "tensor index %zu out of range", i);
    fill_meta(m->plan.index.tensors[i], out);
  });
}

int kk_placements(kk_model* m, const char* tensor, kk_placement* out, size_t cap, size_t* n) {
  return guard([&] {
    need(m, "model");
    need(tensor, "tensor");
    const auto& T = m->plan.index.tensors;
    size_t ti = T.size();
    for (size_t i = 0; i < T.size(); ++i)
      if (T[i].name == tensor) { ti = i; break; }
    if (ti == T.size()) kk::fail(KK_ENOENT, "tensor \"%s\" not in this model", tensor);
    const size_t nl = m->dev_idx.size();
    if (n) *n = nl;
    if (!out) return;
    if (cap < nl) kk::fail(KK_ERANGE, "need room for %zu placements", nl);
    for (size_t li = 0; li < nl; ++li) {
      const kk::Placement& p = m->plan.placement_of_part(m->local_parts[li])[ti];
      kk_placement& o = out[li];
      memset(&o, 0, sizeof o);
      o.device = m->ctx->devs[(size_t)m->dev_idx[li]].ordinal;
      o.dtype = p.dtype;
      o.pool_offset = p.pool_offset;
      o.nbytes = p.nbytes;
      o.n_dims = (uint32_t)p.shape.size();
      for (size_t d = 0; d < p.shape.size(); ++d) o.shape[d] = p.shape[d];
      o.slice_dim = p.slice_dim;
      o.slice_begin = p.slice_begin;
    }
  });
}

int kk_export_size(kk_model* m, int device, size_t* required) {
  return guard([&] {
    need(m, "model");
    need(required, "required");
    int li = kk::model_local_device(m, device);
    *required = kk::model_manifest(m, li).size() + 1;
  });
}

int kk_export(kk_model* m, int device, void* ipc_handle_64B, char* manifest_json, size_t cap) {
  return guard([&] {
    need(m, "model");
    int li = kk::model_local_device(m, device);
    if (manifest_json) {
      std::string s = kk::model_manifest(m, li);
      if (s.size() + 1 > cap) kk::fail(KK_ERANGE, "manifest needs %zu bytes", s.size() + 1);
      memcpy(manifest_json, s.c_str(), s.size() + 1);
    }
    if (ipc_handle_64B) {
      const kk::Pool& pool = m->pools[(size_t)li];
      if (pool.is_nvls()) kk::fail(KK_EUNSUPPORTED, "pools of a KK_FANOUT_NVLS model are VMM allocations: there is no cudaIpcMemHandle for them (export the manifest only, or load with KK_FANOUT_P2P)");
      if (pool.vmm) kk::fail(KK_EUNSUPPORTED, "pools of a KK_CFG_VMM_POOLS context are VMM allocations: there is no cudaIpcMemHandle for them, export the file descriptor (kk_export_fd)");
      kk::model_pool_ipc_handle(m, li, ipc_handle_64B);
    }
  });
}

struct kk_import {
  kk::VmmImport im;
};

int kk_export_fd(kk_model* m, int device, int* fd_out, uint64_t* mapped_bytes) {
  return guard([&] {
    need(m, "model");
    need(fd_out, "fd_out");
    *fd_out = -1;
    int li = kk::model_local_device(m, device);
    const kk::VmmAlloc* vmm = m->pools[(size_t)li].vmm.get();
    if (!vmm) kk::fail(KK_EUNSUPPORTED, "this pool is a cudaMalloc allocation: open the context with KK_CFG_VMM_POOLS to export file descriptors");
    *fd_out = vmm->export_fd();
    if (mapped_bytes) *mapped_bytes = vmm->bytes();
  });
}

int kk_import_fd(int fd, int device, uint64_t mapped_bytes, uint32_t flags, void** dev_ptr, kk_import** out) {
  return guard([&] {
    need(dev_ptr, "dev_ptr");
    need(out, "out");
    *dev_ptr = nullptr;
    *out = nullptr;
    if (fd < 0 || mapped_bytes == 0) kk::fail(KK_EINVAL, "bad fd / size");
    if (flags & ~KK_IMPORT_READONLY) kk::fail(KK_EINVAL, "unknown import flags 0x%x", flags);
    kk_import* im = new kk_import{kk::vmm_import_fd(fd, device, mapped_bytes, (flags & KK_IMPORT_READONLY) != 0)};
    *dev_ptr = im->im.map.ptr();
    *out = im;
  });
}

int kk_import_close(kk_import* im) {
  return guard([&] {
    need(im, "import");
    delete im;
  });
}

int kk_pool_ptr(kk_model* m, int device, void** p, uint64_t* nbytes) {
  return guard([&] {
    need(m, "model");
    int li = kk::model_local_device(m, device);
    if (p) *p = m->pools[(size_t)li].ptr;
    if (nbytes) *nbytes = m->pools[(size_t)li].bytes;
  });
}

int kk_acquire(kk_model* m) {
  return guard([&] {
    need(m, "model");
    std::lock_guard<std::mutex> g(m->ctx->mu);
    if (m->refcount <= 0) kk::fail(KK_ESTATE, "acquire on a released model");
    m->refcount++;
  });
}

int kk_release(kk_model* m) {
  return guard([&] {
    need(m, "model");
    kk::model_release(m);
  });
}

int kk_stats(kk_model* m, char* json, size_t cap) {
  return guard([&] {
    need(m, "model");
    need(json, "json");
    std::string s = kk::model_stats(m);
    if (s.size() + 1 > cap) kk::fail(KK_ERANGE, "stats need %zu bytes", s.size() + 1);
    memcpy(json, s.c_str(), s.size() + 1);
  });
}

int kk_read(kk_model* m, int device, uint64_t off, uint64_t nbytes, void* host_dst) {
  return guard([&] {
    need(m, "model");
    int li = kk::model_local_device(m, device);
    if (nbytes == 0) return;
    need(host_dst, "host_dst");
    const kk::Pool& pool = m->pools[(size_t)li];
    if (off > pool.bytes || nbytes > pool.bytes - off) kk::fail(KK_EINVAL, "range outside the pool");
    KK_CUDA(cudaSetDevice(device));
    KK_CUDA(cudaMemcpy(host_dst, pool.ptr + off, nbytes, cudaMemcpyDeviceToHost));
  });
}

int kk_checksum(kk_model* m, int device, uint64_t off, uint64_t nbytes, uint64_t* out) {
  return guard([&] {
    need(m, "model");
    need(out, "out");
    int li = kk::model_local_device(m, device);
    const kk::Pool& pool = m->pools[(size_t)li];
    if (off > pool.bytes || nbytes > pool.bytes - off) kk::fail(KK_EINVAL, "range outside the pool");
    if (off % 8) kk::fail(KK_EINVAL, "pool_offset must be a multiple of 8");
    kk::Device& d = m->ctx->devs[(size_t)m->dev_idx[(size_t)li]];
    KK_CUDA(cudaSetDevice(device));
    // the accumulator lives in the device's scratch words: a cudaMalloc + cudaFree pair per call synchronises the whole device and, next to a
    // 16 GB pool, stalls for tens of milliseconds every few calls
    std::lock_guard<std::mutex> one(*d.sum_mu);
    unsigned long long* acc = (unsigned long long*)(d.sched.get<uint32_t>() + 32);
    KK_CUDA(cudaMemsetAsync(acc, 0, 8, d.stream));
    KK_CUDA(kk::launch_checksum(pool.ptr + off, nbytes, acc, d.sm_count, d.stream));
    unsigned long long h = 0;
    KK_CUDA(cudaMemcpyAsync(&h, acc, 8, cudaMemcpyDeviceToHost, d.stream));
    KK_CUDA(cudaStreamSynchronize(d.stream));
    *out = h;
  });
}

int kk_stage_resident(kk_model* m) {
  return guard([&] {
    need(m, "model");
    kk::model_stage_resident(m);
  });
}

int kk_convert_resident(kk_model* m, float* ms_total, float* ms_per_launch, size_t cap, size_t* n_launches) {
  return guard([&] {
    need(m, "model");
    kk::model_convert_resident(m, ms_total, ms_per_launch, cap, n_launches);
  });
}

int kk_unstage_resident(kk_model* m) {
  return guard([&] {
    need(m, "model");
    kk::model_unstage_resident(m);
  });
}

int kk_probe_hbm(kk_ctx* ctx, int device, int kind, uint64_t nbytes, float* ms) {
  return guard([&] {
    need(ctx, "ctx");
    need(ms, "ms");
    *ms = 0.f;
    if (kind != KK_PROBE_WRITE && kind != KK_PROBE_COPY) kk::fail(KK_EINVAL, "unknown probe kind %d", kind);
    kk::Device* d = nullptr;
    for (auto& x : ctx->devs)
      if (x.ordinal == device) d = &x;
    if (!d) kk::fail(KK_EINVAL, "device %d is not part of this context", device);
    nbytes &= ~(uint64_t)15;
    if (nbytes == 0) kk::fail(KK_EINVAL, "probe needs at least 16 bytes");
    kk::DevBuf dst(device, nbytes, "the probe"), src;
    if (kind == KK_PROBE_COPY) {
      src = kk::DevBuf(device, nbytes, "the probe");
      KK_CUDA(cudaMemsetAsync(src.get(), 0x3C, nbytes, d->stream));
    }
    kk::EventSet ev(2);
    ev.create_all();
    for (int pass = 0; pass < 2; ++pass) {  // pass 0 warms up (first touch of the scratch pages), pass 1 is timed
      if (pass) KK_CUDA(cudaEventRecord(ev[0], d->stream));
      if (kind == KK_PROBE_WRITE) KK_CUDA(kk::launch_fill(dst.get(), nbytes, d->sm_count, d->stream));
      else KK_CUDA(kk::launch_ldg_copy(src.get(), dst.get(), nbytes, d->sm_count, d->stream));
      if (pass) KK_CUDA(cudaEventRecord(ev[1], d->stream));
    }
    KK_CUDA(cudaStreamSynchronize(d->stream));
    KK_CUDA(cudaEventElapsedTime(ms, ev[0], ev[1]));
  });
}

int kk_device_identity(int device, char* pci_bus_id, size_t pci_cap, char* uuid, size_t uuid_cap) {
  return guard([&] {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess) { cudaGetLastError(); kk::fail(KK_ECUDA, "no usable CUDA device"); }
    if (device < 0 || device >= count) kk::fail(KK_EINVAL, "device %d out of range (0..%d)", device, count - 1);
    if (pci_bus_id && pci_cap < 16) kk::fail(KK_ERANGE, "pci_bus_id needs 16 bytes");
    if (uuid && uuid_cap < 41) kk::fail(KK_ERANGE, "uuid needs 41 bytes");
    kk::device_identity(device, pci_bus_id, pci_cap, uuid, uuid_cap);
  });
}

int kk_probe_peer(kk_model* m, int rank, int which, uint64_t* nbytes, float* ms) {
  return guard([&] {
    need(m, "model");
    need(nbytes, "nbytes");
    need(ms, "ms");
    *ms = 0.f;
    kk::PeerKind kind;
    bool by_ptr;
    if (!buf_kind(which, kind, by_ptr) || by_ptr) kk::fail(KK_EINVAL, "probe: buffer kind %d (KK_BUF_POOL, KK_BUF_RAW or KK_BUF_SLICE)", which);
    kk::model_probe_peer(m, rank, kind, *nbytes, ms);
  });
}

}  // extern "C"
#pragma GCC visibility pop
