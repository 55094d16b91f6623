// Device memory the library owns: cudaMalloc buffers (DevBuf), VMM allocations exported as a POSIX file descriptor and mapped by another
// process READ-ONLY (KK_CFG_VMM_POOLS), and per-device VMM allocations bound to one NVSwitch multicast object (KK_FANOUT_NVLS).  See kk_mem.cpp.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <utility>
#include <vector>

#include "kk_common.hpp"

namespace kk {

#define KK_CUDA(expr)                                                                               \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) ::kk::fail(KK_ECUDA, "%s: %s (%s)", #expr, cudaGetErrorString(_e), cudaGetErrorName(_e)); \
  } while (0)

// One cudaMalloc allocation and the device it lives on.  Move-only; the destructor frees it on that device and never throws.
class DevBuf {
 public:
  DevBuf() = default;
  // `bytes` on device `ordinal`, which is made current.  KK_ENOMEM naming the device, the size and `what` the buffer is for.
  DevBuf(int ordinal, uint64_t bytes, const char* what);
  ~DevBuf();
  DevBuf(DevBuf&& o) noexcept { swap(o); }
  DevBuf& operator=(DevBuf&& o) noexcept {
    DevBuf t(std::move(o));
    swap(t);
    return *this;
  }
  template <class T = uint8_t>
  T* get() const { return reinterpret_cast<T*>(p_); }
  uint64_t bytes() const { return bytes_; }
  explicit operator bool() const { return p_ != nullptr; }

 private:
  void swap(DevBuf& o) noexcept {
    std::swap(p_, o.p_);
    std::swap(bytes_, o.bytes_);
    std::swap(dev_, o.dev_);
  }
  uint8_t* p_ = nullptr;
  uint64_t bytes_ = 0;
  int dev_ = -1;
};

// A physical allocation or multicast object handle, released when the owner goes.
struct MemHandle {
  CUmemGenericAllocationHandle h = 0;
  MemHandle() = default;
  ~MemHandle();
  MemHandle(MemHandle&& o) noexcept : h(std::exchange(o.h, 0)) {}
};

// A reserved address range with an allocation mapped over it and access granted (cuMemAddressReserve -> cuMemMap -> cuMemSetAccess), undone
// in reverse when the owner goes.  `feature` and `which` name the mapping in error messages.
class Mapping {
 public:
  Mapping() = default;
  Mapping(const char* feature, const char* which, CUmemGenericAllocationHandle h, size_t size, size_t align, const std::vector<CUmemAccessDesc>& access);
  ~Mapping();
  Mapping(Mapping&& o) noexcept : va_(std::exchange(o.va_, 0)), size_(o.size_), mapped_(std::exchange(o.mapped_, false)) {}
  Mapping& operator=(Mapping&& o) noexcept {
    Mapping t(std::move(o));
    std::swap(va_, t.va_);
    std::swap(size_, t.size_);
    std::swap(mapped_, t.mapped_);
    return *this;
  }
  uint8_t* ptr() const { return reinterpret_cast<uint8_t*>(va_); }

 private:
  CUdeviceptr va_ = 0;
  size_t size_ = 0;
  bool mapped_ = false;
};

// One physical allocation on one device, mapped read-write into this process for `access` devices.
class VmmAlloc {
 public:
  // >= bytes on CUDA device `ordinal`, exportable as a POSIX fd; read-write for every device in `access` (the owner is always included).
  // Throws kk::Error (KK_EUNSUPPORTED when the driver lacks VMM / fd handles, KK_ENOMEM, KK_ECUDA).
  void create(int ordinal, uint64_t bytes, const std::vector<int>& access);
  uint8_t* ptr() const { return map_.ptr(); }
  uint64_t bytes() const { return size_; }
  // A new file descriptor referring to the allocation (the caller owns and closes it).  Whoever holds it can map the memory with the
  // protection it chooses — hand it only to processes that may at least read the weights; kk_import_fd maps it read-only.
  int export_fd() const;

 private:
  MemHandle handle_;
  Mapping map_;  // declared after the handle: unmapped before the handle is released
  uint64_t size_ = 0;
};

// Consumer side: an exported allocation mapped into this process on `ordinal` (readonly = CU_MEM_ACCESS_FLAGS_PROT_READ).  Unmapped and
// released when the owner goes.
struct VmmImport {
  MemHandle handle;
  Mapping map;
};
VmmImport vmm_import_fd(int fd, int ordinal, uint64_t bytes, bool readonly);

// NVLS pools: one allocation per device, all bound to one multicast object.
class NvlsPools {
 public:
  NvlsPools() = default;
  ~NvlsPools();
  NvlsPools(const NvlsPools&) = delete;
  NvlsPools& operator=(const NvlsPools&) = delete;

  // Every listed device reports CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED and the driver exports the multicast entry points.
  static bool supported(const std::vector<int>& ordinals, std::string* why);
  // One allocation of >= bytes on every device, all bound at offset 0 of one multicast object, all mapped.  Throws kk::Error
  // (KK_EUNSUPPORTED when the host does not expose NVLS, KK_ENOMEM, KK_ECUDA); a partially built object cleans up in its destructor.
  void create(const std::vector<int>& ordinals, uint64_t bytes);

  uint8_t* pool(size_t i) const { return uc_[i].ptr(); }  // unicast address of device i's allocation (readable / writable from every device)
  uint8_t* multicast() const { return mc_map_.ptr(); }    // multicast address: a multimem.st here lands at the same offset of every pool

 private:
  size_t size_ = 0;  // of each allocation after rounding to the multicast granularity
  std::vector<CUdevice> devs_;
  MemHandle mc_;
  std::vector<MemHandle> mem_;  // one physical allocation per device
  size_t n_bound_ = 0;          // mem_[0, n_bound_) are bound to mc_
  std::vector<Mapping> uc_;     // unicast mapping of each device's allocation (accessible from every device)
  Mapping mc_map_;
};

}  // namespace kk
