// NVLS (NVLink SHARP) substrate, host side: a VMM-backed symmetric heap with an NVSwitch multicast mapping, on which the switch
// does the arithmetic — `multimem.ld_reduce` (one load returns the sum over every GPU's copy) and `multimem.st` (one store lands in
// every GPU's copy).
//
//   cudaIpc heap (comm.cu)           every byte a rank reduces crosses ITS link once per peer:  (F-1)/F · B inbound
//   multicast heap (this file)       the switch adds the F copies and returns one:                   1/F · B inbound
//
// All through driver entry points resolved at run time — nothing links against libcuda:
//   pb_vmm_create / export fd → peers import → pb_vmm_map          physical allocation shared by POSIX file descriptor
//   pb_mc_create (rank 0) → fd to peers → pb_mc_add_device (all) → pb_mc_bind (all) → pb_vmm_map(mc handle)
// The fd exchange itself is SCM_RIGHTS over Unix sockets and lives in Python (parallel/multicast.py).
//
// The kernels that use the multicast mapping are in comm.cu, next to the flag wait they share: the multimem barrier and
// all-reduce (pb_mc_all_reduce), the gradient reduce-scatter (pb_grad_reduce with mc_grads) and adamw_push's parameter publish.
// Summation order inside the switch is fixed by the hardware, not by rank order: results are deterministic for a given
// topology but NOT bitwise equal to the peer-load path, which is why the engine keeps this opt-in (PB_NVLS=1).
#include <cuda.h>

#include <mutex>

#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------ driver entry points
struct Driver {
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*MemExport)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
  CUresult (*MemImport)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*MemGetGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*McCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
  CUresult (*McAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
  CUresult (*McBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long) = nullptr;
  CUresult (*McUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t) = nullptr;
  CUresult (*McGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
  CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  bool ok = false;
};

template <typename F>
bool resolve(F& fn, const char* name) {
  void* sym = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &sym, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return false;
  fn = reinterpret_cast<F>(sym);
  return true;
}

const Driver& driver() {
  static Driver d;
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFree(nullptr);  // bind the primary context on this thread before touching the driver API
    d.ok = resolve(d.MemCreate, "cuMemCreate") && resolve(d.MemRelease, "cuMemRelease") &&
           resolve(d.MemExport, "cuMemExportToShareableHandle") && resolve(d.MemImport, "cuMemImportFromShareableHandle") &&
           resolve(d.MemAddressReserve, "cuMemAddressReserve") && resolve(d.MemAddressFree, "cuMemAddressFree") &&
           resolve(d.MemMap, "cuMemMap") && resolve(d.MemUnmap, "cuMemUnmap") && resolve(d.MemSetAccess, "cuMemSetAccess") &&
           resolve(d.MemGetGranularity, "cuMemGetAllocationGranularity") && resolve(d.McCreate, "cuMulticastCreate") &&
           resolve(d.McAddDevice, "cuMulticastAddDevice") && resolve(d.McBindMem, "cuMulticastBindMem") &&
           resolve(d.McUnbind, "cuMulticastUnbind") && resolve(d.McGetGranularity, "cuMulticastGetGranularity") &&
           resolve(d.DeviceGet, "cuDeviceGet") && resolve(d.DeviceGetAttribute, "cuDeviceGetAttribute");
  });
  return d;
}

constexpr int kNoDriver = -10;
inline int rc(CUresult r) { return r == CUDA_SUCCESS ? 0 : -100 - (int)r; }  // -100-CUresult: distinguishable from cudaError_t

CUmemAllocationProp device_prop(int dev) {
  CUmemAllocationProp p = {};
  p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  p.location.id = dev;
  p.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return p;
}

CUmulticastObjectProp mc_prop(int ndev, size_t size) {
  CUmulticastObjectProp p = {};
  p.numDevices = (unsigned)ndev;
  p.size = size;
  p.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return p;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ host API (C ABI)
// 1 = this device can join a multicast object (NVSwitch + driver support), 0 = no, <0 = error.
PB_EXPORT int pb_mc_supported(int dev) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  CUdevice cd;
  if (int e = rc(d.DeviceGet(&cd, dev))) return e;
  int v = 0;
  if (int e = rc(d.DeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cd))) return e;
  return v ? 1 : 0;
}

// Size granularity that satisfies BOTH the physical allocation and (when ndev > 1) the multicast binding.
PB_EXPORT int pb_vmm_granularity(int dev, int ndev, size_t size, size_t* out) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  CUmemAllocationProp p = device_prop(dev);
  size_t g = 0, gm = 0;
  if (int e = rc(d.MemGetGranularity(&g, &p, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED))) return e;
  if (ndev > 1) {
    CUmulticastObjectProp mp = mc_prop(ndev, size);
    if (int e = rc(d.McGetGranularity(&gm, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED))) return e;
  }
  *out = g > gm ? g : gm;
  return 0;
}

PB_EXPORT int pb_vmm_create(int dev, size_t size, uint64_t* handle, int* fd) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  CUmemAllocationProp p = device_prop(dev);
  CUmemGenericAllocationHandle h;
  if (int e = rc(d.MemCreate(&h, size, &p, 0))) return e;
  int out_fd = -1;
  if (int e = rc(d.MemExport(&out_fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0))) {
    d.MemRelease(h);
    return e;
  }
  *handle = (uint64_t)h;
  *fd = out_fd;
  return 0;
}

// Works for physical allocations and for multicast objects alike (both are generic allocation handles).
PB_EXPORT int pb_vmm_import(int fd, uint64_t* handle) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  CUmemGenericAllocationHandle h;
  if (int e = rc(d.MemImport(&h, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR))) return e;
  *handle = (uint64_t)h;
  return 0;
}

// Reserve a VA range, map `handle` into it and give `dev` read/write access.
PB_EXPORT int pb_vmm_map(uint64_t handle, size_t size, size_t align, int dev, void** ptr) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  CUdeviceptr va = 0;
  if (int e = rc(d.MemAddressReserve(&va, size, align, 0, 0))) return e;
  if (int e = rc(d.MemMap(va, size, 0, (CUmemGenericAllocationHandle)handle, 0))) {
    d.MemAddressFree(va, size);
    return e;
  }
  CUmemAccessDesc acc = {};
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = dev;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  if (int e = rc(d.MemSetAccess(va, size, &acc, 1))) {
    d.MemUnmap(va, size);
    d.MemAddressFree(va, size);
    return e;
  }
  *ptr = (void*)va;
  return 0;
}

PB_EXPORT int pb_vmm_unmap(void* ptr, size_t size) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  if (int e = rc(d.MemUnmap((CUdeviceptr)ptr, size))) return e;
  return rc(d.MemAddressFree((CUdeviceptr)ptr, size));
}

PB_EXPORT int pb_vmm_release(uint64_t handle) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  return rc(d.MemRelease((CUmemGenericAllocationHandle)handle));
}

PB_EXPORT int pb_mc_create(int ndev, size_t size, uint64_t* handle, int* fd) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  CUmulticastObjectProp p = mc_prop(ndev, size);
  CUmemGenericAllocationHandle h;
  if (int e = rc(d.McCreate(&h, &p))) return e;
  int out_fd = -1;
  if (int e = rc(d.MemExport(&out_fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0))) {
    d.MemRelease(h);
    return e;
  }
  *handle = (uint64_t)h;
  *fd = out_fd;
  return 0;
}

PB_EXPORT int pb_mc_add_device(uint64_t mc, int dev) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  CUdevice cd;
  if (int e = rc(d.DeviceGet(&cd, dev))) return e;
  return rc(d.McAddDevice((CUmemGenericAllocationHandle)mc, cd));
}

// Every device must have been added (by every process) before the first bind: the caller barriers in between.
PB_EXPORT int pb_mc_bind(uint64_t mc, uint64_t mem, size_t size) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  return rc(d.McBindMem((CUmemGenericAllocationHandle)mc, 0, (CUmemGenericAllocationHandle)mem, 0, size, 0));
}

PB_EXPORT int pb_mc_unbind(uint64_t mc, int dev, size_t size) {
  const Driver& d = driver();
  if (!d.ok) return kNoDriver;
  CUdevice cd;
  if (int e = rc(d.DeviceGet(&cd, dev))) return e;
  return rc(d.McUnbind((CUmemGenericAllocationHandle)mc, cd, 0, size));
}
