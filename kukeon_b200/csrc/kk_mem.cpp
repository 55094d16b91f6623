// Device memory the library owns.
//
// Every staging buffer, segment table, image and default pool is a cudaMalloc allocation held by a DevBuf.  The rest goes through the driver's
// virtual-memory-management and multicast entry points, fetched at run time with cudaGetDriverEntryPoint: the library keeps linking only the
// static runtime and still loads on a machine without libcuda (the CPU test tier checks exactly that).
//
// VMM pools (KK_CFG_VMM_POOLS).  Why they exist: a cudaIpcMemHandle maps the exporter's memory READ-WRITE in every process that opens it, so
// handing the pool's IPC handle to N agent containers lets any one of them overwrite the weights the other N-1 read (round-1 review; the unit
// of isolation of the orchestrator is the cell).  Memory created with cuMemCreate + CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR is shared as a
// file descriptor instead, and the importer's mapping carries the protection given to cuMemSetAccess: kk_import_fd maps it with
// CU_MEM_ACCESS_FLAGS_PROT_READ, a store through that mapping faults in the importing process and never reaches the pool.
//
// NVLS (NVSwitch multicast) pools for KK_FANOUT_NVLS: one physical allocation per device bound to one multicast object, so that a single
// multimem.st from the convert kernel lands in every device's pool.  One process owning all devices only; pools allocated this way cannot be
// exported with cudaIpcGetMemHandle (they are VMM allocations), which is why this path is the comparison the north_star names, not the
// default (DESIGN.md §3.1).
#include "kk_mem.hpp"

#include <algorithm>
#include <cstring>
#include <type_traits>

namespace kk {

DevBuf::DevBuf(int ordinal, uint64_t bytes, const char* what) : dev_(ordinal) {
  KK_CUDA(cudaSetDevice(ordinal));
  const cudaError_t e = cudaMalloc((void**)&p_, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    p_ = nullptr;
    fail(KK_ENOMEM, "device %d: cudaMalloc(%llu) for %s failed: %s", ordinal, (unsigned long long)bytes, what, cudaGetErrorString(e));
  }
  bytes_ = bytes;
}

DevBuf::~DevBuf() {
  if (!p_) return;
  cudaSetDevice(dev_);
  cudaFree(p_);
  cudaGetLastError();  // a failed free must not surface as the error of the next, unrelated call
}

namespace {

const char kVmm[] = "VMM pools";
const char kNvls[] = "fan-out NVLS";

struct Drv {
  // virtual memory management: VMM pools and NVLS
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
  CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
  // multicast: NVLS only, so that a driver without it still gives working VMM pools
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long) = nullptr;
  CUresult (*MulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t) = nullptr;
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
  const char* missing = nullptr;     // first entry point of the first group the driver does not export
  const char* missing_mc = nullptr;  // first multicast entry point it does not export
};

const Drv& entry_points() {
  static const Drv d = [] {
    Drv x;
    auto get = [](auto& fn, const char* name, const char*& missing) {
      void* p = nullptr;
      cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
      if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
        cudaGetLastError();
        p = nullptr;
        if (!missing) missing = name;
      }
      fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(p);
    };
    get(x.MemCreate, "cuMemCreate", x.missing);
    get(x.MemRelease, "cuMemRelease", x.missing);
    get(x.MemAddressReserve, "cuMemAddressReserve", x.missing);
    get(x.MemAddressFree, "cuMemAddressFree", x.missing);
    get(x.MemMap, "cuMemMap", x.missing);
    get(x.MemUnmap, "cuMemUnmap", x.missing);
    get(x.MemSetAccess, "cuMemSetAccess", x.missing);
    get(x.MemGetAllocationGranularity, "cuMemGetAllocationGranularity", x.missing);
    get(x.MemExportToShareableHandle, "cuMemExportToShareableHandle", x.missing);
    get(x.MemImportFromShareableHandle, "cuMemImportFromShareableHandle", x.missing);
    get(x.DeviceGet, "cuDeviceGet", x.missing);
    get(x.DeviceGetAttribute, "cuDeviceGetAttribute", x.missing);
    get(x.GetErrorString, "cuGetErrorString", x.missing);
    get(x.MulticastCreate, "cuMulticastCreate", x.missing_mc);
    get(x.MulticastAddDevice, "cuMulticastAddDevice", x.missing_mc);
    get(x.MulticastBindMem, "cuMulticastBindMem", x.missing_mc);
    get(x.MulticastUnbind, "cuMulticastUnbind", x.missing_mc);
    get(x.MulticastGetGranularity, "cuMulticastGetGranularity", x.missing_mc);
    return x;
  }();
  return d;
}

// The entry points `feature` needs (with multicast: NVLS's as well); KK_EUNSUPPORTED naming the first one the driver does not export.
const Drv& drv(const char* feature, bool multicast = false) {
  const Drv& d = entry_points();
  const char* missing = d.missing ? d.missing : multicast ? d.missing_mc : nullptr;
  if (missing) fail(KK_EUNSUPPORTED, "%s: the CUDA driver does not export %s", feature, missing);
  return d;
}

void check(const char* feature, CUresult r, const char* what) {
  if (r == CUDA_SUCCESS) return;
  const char* s = nullptr;
  entry_points().GetErrorString(r, &s);
  // NOT_SUPPORTED / NOT_PERMITTED / SYSTEM_NOT_READY mean "this host does not offer it (right now)", not a bug on our side
  const int code = (r == CUDA_ERROR_NOT_SUPPORTED || r == CUDA_ERROR_NOT_PERMITTED || r == CUDA_ERROR_SYSTEM_NOT_READY) ? KK_EUNSUPPORTED
                   : r == CUDA_ERROR_OUT_OF_MEMORY ? KK_ENOMEM : KK_ECUDA;
  fail(code, "%s: %s: %s (%d)", feature, what, s ? s : "?", (int)r);
}

// The driver calls below want the device's primary context current on the calling thread.
void make_current(const char* who, int ordinal) {
  if (cudaSetDevice(ordinal) != cudaSuccess) { cudaGetLastError(); fail(KK_ECUDA, "%s: cudaSetDevice(%d)", who, ordinal); }
  cudaFree(nullptr);
}

CUmemAllocationProp prop_for(int ordinal, CUmemAllocationHandleType handles) {
  CUmemAllocationProp ap;
  memset(&ap, 0, sizeof ap);
  ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  ap.location.id = ordinal;
  ap.requestedHandleTypes = handles;
  return ap;
}

size_t granularity(const char* feature, const CUmemAllocationProp& ap) {
  size_t g = 0;
  check(feature, entry_points().MemGetAllocationGranularity(&g, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED), "cuMemGetAllocationGranularity");
  return g ? g : (size_t)(2u << 20);
}

CUmemAccessDesc access_desc(int ordinal, CUmemAccess_flags flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE) {
  CUmemAccessDesc a;
  memset(&a, 0, sizeof a);
  a.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  a.location.id = ordinal;
  a.flags = flags;
  return a;
}

}  // namespace

MemHandle::~MemHandle() {
  if (h) entry_points().MemRelease(h);
}

// Delegates to the default constructor so that the destructor runs, and undoes what was done, when a step below throws.
Mapping::Mapping(const char* feature, const char* which, CUmemGenericAllocationHandle h, size_t size, size_t align,
                 const std::vector<CUmemAccessDesc>& access)
    : Mapping() {
  const Drv& d = entry_points();
  const std::string w(which);
  CUdeviceptr va = 0;
  check(feature, d.MemAddressReserve(&va, size, align, 0, 0), ("cuMemAddressReserve" + w).c_str());
  va_ = va;
  size_ = size;
  check(feature, d.MemMap(va_, size, 0, h, 0), ("cuMemMap" + w).c_str());
  mapped_ = true;
  check(feature, d.MemSetAccess(va_, size, access.data(), access.size()), ("cuMemSetAccess" + w).c_str());
}

Mapping::~Mapping() {
  if (!va_) return;
  const Drv& d = entry_points();
  if (mapped_) d.MemUnmap(va_, size_);
  d.MemAddressFree(va_, size_);
}

void VmmAlloc::create(int ordinal, uint64_t bytes, const std::vector<int>& access) {
  const Drv& d = drv(kVmm);  // a missing entry point is KK_EUNSUPPORTED before anything is allocated
  make_current(kVmm, ordinal);
  const CUmemAllocationProp ap = prop_for(ordinal, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
  const size_t gran = granularity(kVmm, ap);
  size_ = (bytes + gran - 1) / gran * gran;
  if (size_ == 0) size_ = gran;
  check(kVmm, d.MemCreate(&handle_.h, (size_t)size_, &ap, 0), "cuMemCreate");
  std::vector<CUmemAccessDesc> acc{access_desc(ordinal)};
  for (int o : access)
    if (std::none_of(acc.begin(), acc.end(), [&](const CUmemAccessDesc& a) { return a.location.id == o; })) acc.push_back(access_desc(o));
  map_ = Mapping(kVmm, "", handle_.h, (size_t)size_, gran, acc);
}

int VmmAlloc::export_fd() const {
  if (!handle_.h) fail(KK_ESTATE, "VMM pools: nothing allocated");
  int fd = -1;
  check(kVmm, entry_points().MemExportToShareableHandle(&fd, handle_.h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0), "cuMemExportToShareableHandle");
  return fd;
}

VmmImport vmm_import_fd(int fd, int ordinal, uint64_t bytes, bool readonly) {
  const Drv& d = drv(kVmm);
  make_current("VMM import", ordinal);
  const CUmemAllocationProp ap = prop_for(ordinal, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
  const size_t gran = granularity(kVmm, ap);
  VmmImport im;
  check(kVmm, d.MemImportFromShareableHandle(&im.handle.h, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR), "cuMemImportFromShareableHandle");
  im.map = Mapping(kVmm, " (is `bytes` the exported size?)", im.handle.h, (size_t)((bytes + gran - 1) / gran * gran), gran,
                   {access_desc(ordinal, readonly ? CU_MEM_ACCESS_FLAGS_PROT_READ : CU_MEM_ACCESS_FLAGS_PROT_READWRITE)});
  return im;
}

NvlsPools::~NvlsPools() {
  // reverse order of creation: the mappings, the bindings, then (as members) the allocations and the multicast object
  mc_map_ = Mapping();
  uc_.clear();
  for (size_t i = 0; i < n_bound_; ++i) entry_points().MulticastUnbind(mc_.h, devs_[i], 0, size_);
}

bool NvlsPools::supported(const std::vector<int>& ordinals, std::string* why) {
  try {
    const Drv& d = drv(kNvls, true);
    for (int o : ordinals) {
      CUdevice dev;
      check(kNvls, d.DeviceGet(&dev, o), "cuDeviceGet");
      int v = 0;
      check(kNvls, d.DeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev), "cuDeviceGetAttribute(MULTICAST_SUPPORTED)");
      if (!v) {
        if (why) *why = "device " + std::to_string(o) + " does not support multicast (no NVSwitch / NVLS on this host)";
        return false;
      }
    }
    return true;
  } catch (const Error& e) {
    if (why) *why = e.what();
    return false;
  }
}

void NvlsPools::create(const std::vector<int>& ordinals, uint64_t bytes) {
  const Drv& d = drv(kNvls, true);
  const size_t n = ordinals.size();
  if (n < 2) fail(KK_EINVAL, "fan-out NVLS needs at least two devices");
  devs_.resize(n);
  for (size_t i = 0; i < n; ++i) check(kNvls, d.DeviceGet(&devs_[i], ordinals[i]), "cuDeviceGet");

  CUmulticastObjectProp mp;
  memset(&mp, 0, sizeof mp);
  mp.numDevices = (unsigned)n;
  mp.handleTypes = 0;  // not shared with other processes
  mp.flags = 0;
  mp.size = (size_t)bytes;
  size_t gran = 0;
  check(kNvls, d.MulticastGetGranularity(&gran, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED), "cuMulticastGetGranularity");
  CUmemAllocationProp ap = prop_for(ordinals[0], CU_MEM_HANDLE_TYPE_NONE);
  gran = std::max(gran, granularity(kNvls, ap));
  size_ = (size_t)((bytes + gran - 1) / gran * gran);
  mp.size = size_;

  check(kNvls, d.MulticastCreate(&mc_.h, &mp), "cuMulticastCreate");
  for (size_t i = 0; i < n; ++i) check(kNvls, d.MulticastAddDevice(mc_.h, devs_[i]), "cuMulticastAddDevice");  // all devices before any bind

  std::vector<CUmemAccessDesc> acc;
  for (int o : ordinals) acc.push_back(access_desc(o));
  mem_.resize(n);
  for (size_t i = 0; i < n; ++i) {
    ap.location.id = ordinals[i];
    check(kNvls, d.MemCreate(&mem_[i].h, size_, &ap, 0), "cuMemCreate");
    check(kNvls, d.MulticastBindMem(mc_.h, 0, mem_[i].h, 0, size_, 0), "cuMulticastBindMem");
    n_bound_ = i + 1;
    uc_.push_back(Mapping(kNvls, "", mem_[i].h, size_, gran, acc));
  }
  mc_map_ = Mapping(kNvls, "(multicast)", mc_.h, size_, gran, acc);
}

}  // namespace kk
