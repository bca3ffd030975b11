// NVLS (NVLink SHARP) substrate: a VMM-backed symmetric heap with an NVSwitch multicast mapping, and the kernels that let
// the switch do the arithmetic — `multimem.ld_reduce` (one load returns the sum over every GPU's copy) and `multimem.st`
// (one store lands in every GPU's copy).
//
//   cudaIpc heap (comm.cu)           every byte a rank reduces crosses ITS link once per peer:  (F-1)/F · B inbound
//   multicast heap (this file)       the switch adds the F copies and returns one:                   1/F · B inbound
//
// Host side (all through driver entry points resolved at run time — nothing links against libcuda):
//   pb_vmm_create / export fd → peers import → pb_vmm_map          physical allocation shared by POSIX file descriptor
//   pb_mc_create (rank 0) → fd to peers → pb_mc_add_device (all) → pb_mc_bind (all) → pb_vmm_map(mc handle)
// The fd exchange itself is SCM_RIGHTS over Unix sockets and lives in Python (parallel/multicast.py).
//
// Device side:
//   mc_barrier            multimem.red on a flag word: ONE instruction increments the counter on every GPU
//   pb_mc_all_reduce      in place, two-shot in one kernel: rank r reduces slice r through the switch and multicasts it back
//   pb_mc_grad_reduce     drop-in for grad_reduce (comm.cu): out = scale · Σ_peers grad, + Σ out² partials, one switch load
//
// Summation order inside the switch is fixed by the hardware, not by rank order: results are deterministic for a given
// topology but NOT bitwise equal to the peer-load path, which is why the engine keeps this opt-in (PB_NVLS=1).
#include <cuda.h>

#include <mutex>

#include "common.cuh"

using namespace pb;

namespace {

constexpr unsigned long long kMcSpinTimeoutNs = 20ull * 1000ull * 1000ull * 1000ull;

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

// ------------------------------------------------------------------------------------------------ multimem PTX
namespace {

__device__ __forceinline__ float4 mc_ld_reduce_f32x4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void mc_st_f32x4(float* mc, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
// 8 bf16 per access; the switch accumulates in fp32 (.acc::f32) and rounds once.
__device__ __forceinline__ uint4 mc_ld_reduce_bf16x8(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void mc_st_bf16x8(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void mc_red_release_add_u32(uint32_t* mc, uint32_t v) {
  asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// All-ranks barrier for ONE block index: every rank's block `b` adds 1 to flag[b] on every GPU with a single multimem.red,
// then spins on its own copy until `world` arrivals of this phase are in. Counters only grow: phase k of launch `epoch`
// (k = 0 arrive, 1 depart) completes at world·(2·(epoch-1) + k + 1), so no reset and no ABA across launches.
__device__ __forceinline__ void mc_barrier(uint32_t* mc_flags, const uint32_t* local_flags, uint32_t target, uint32_t* err) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    mc_red_release_add_u32(mc_flags + blockIdx.x, 1u);
    const unsigned long long t0 = now_ns();
    while ((int32_t)(ld_acquire_sys(local_flags + blockIdx.x) - target) < 0) {
      __nanosleep(32);
      if (now_ns() - t0 > kMcSpinTimeoutNs) {
        if (err) atomicExch(err, 2u);
        break;
      }
    }
  }
  __syncthreads();
}

// In-place all-reduce over the multicast mapping. n16 = number of 16-byte units; each rank owns a contiguous 1/world of them.
template <bool BF16>
__global__ void __launch_bounds__(512) mc_all_reduce_kernel(void* mc, int64_t n16, uint32_t* mc_flags, const uint32_t* local_flags,
                                                             int rank, int world, uint32_t epoch, uint32_t* err) {
  const uint32_t base = (uint32_t)world * 2u * (epoch - 1u);
  mc_barrier(mc_flags, local_flags, base + (uint32_t)world, err);  // every rank's input is in place
  const int64_t per = (n16 + world - 1) / world;
  const int64_t lo = per * rank, hi = lo + per < n16 ? lo + per : n16;
  uint4* p = reinterpret_cast<uint4*>(mc);
  for (int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (int64_t)gridDim.x * blockDim.x) {
    if constexpr (BF16) {
      const uint4 v = mc_ld_reduce_bf16x8(p + i);
      mc_st_bf16x8(p + i, v);
    } else {
      const float4 v = mc_ld_reduce_f32x4(reinterpret_cast<const float*>(p + i));
      mc_st_f32x4(reinterpret_cast<float*>(p + i), v);
    }
  }
  mc_barrier(mc_flags, local_flags, base + 2u * (uint32_t)world, err);  // every slice has been written everywhere
}

// NVLS form of grad_reduce_kernel (comm.cu): same contract, the peer loop replaced by one switch-side reduction.
__global__ void __launch_bounds__(512) mc_grad_reduce_kernel(const float* __restrict__ mc_grads, int64_t off, int64_t n, float scale,
                                                             float* __restrict__ out, float* __restrict__ sumsq_partial,
                                                             const uint32_t* wait_flags, int slot_base, uint32_t expect, int npeers,
                                                             uint32_t* err) {
  __shared__ float red[32];
  if (wait_flags != nullptr) {
    if ((int)threadIdx.x < npeers) {
      const unsigned long long t0 = now_ns();
      while ((int32_t)(ld_acquire_sys(wait_flags + slot_base + threadIdx.x) - expect) < 0) {
        __nanosleep(64);
        if (now_ns() - t0 > kMcSpinTimeoutNs) {
          if (err) atomicExch(err, 1u);
          break;
        }
      }
    }
    __syncthreads();
  }
  const int64_t nvec = n >> 2;
  float ss = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    float4 acc = mc_ld_reduce_f32x4(mc_grads + off + 4 * i);
    acc.x *= scale, acc.y *= scale, acc.z *= scale, acc.w *= scale;
    reinterpret_cast<float4*>(out)[i] = acc;
    ss += acc.x * acc.x + acc.y * acc.y + acc.z * acc.z + acc.w * acc.w;
  }
  ss = block_sum(ss, red);
  if (threadIdx.x == 0) sumsq_partial[blockIdx.x] += ss;
}

}  // namespace

// Number of flag words an all-reduce needs (one per block) — the grid is fixed so that every rank launches the same one
// and all blocks are co-resident (a spinning block must never wait for a partner that is queued behind it).
PB_EXPORT int pb_mc_all_reduce_grid() { return 132; }

// dtype: 0 = f32, 1 = bf16. `mc_data` and `mc_flags` are addresses in the MULTICAST mapping, `local_flags` the same words
// in this rank's unicast mapping. nbytes must be a multiple of 16. `epoch` starts at 1 and grows by 1 per call on every rank.
PB_EXPORT int pb_mc_all_reduce(void* mc_data, int64_t nbytes, int dtype, uint32_t* mc_flags, const uint32_t* local_flags, int rank,
                               int world, uint32_t epoch, uint32_t* err, cudaStream_t stream) {
  if (nbytes % 16 != 0 || epoch == 0 || world < 1) return -1;
  const int grid = pb_mc_all_reduce_grid();
  if (dtype == 1)
    mc_all_reduce_kernel<true><<<grid, 512, 0, stream>>>(mc_data, nbytes / 16, mc_flags, local_flags, rank, world, epoch, err);
  else if (dtype == 0)
    mc_all_reduce_kernel<false><<<grid, 512, 0, stream>>>(mc_data, nbytes / 16, mc_flags, local_flags, rank, world, epoch, err);
  else
    return -1;
  PB_CHECK_LAUNCH();
  return 0;
}

// Same arguments as pb_grad_reduce, except that the gradients come as ONE multicast address instead of a peer table.
// off and n are in elements; both must be multiples of 4 (they are: shards are SHARD_ALIGN-aligned).
PB_EXPORT int pb_mc_grad_reduce(const float* mc_grads, int64_t off, int64_t n, float scale, float* out, float* sumsq_partial,
                                const uint32_t* wait_flags, int slot_base, uint32_t expect, int npeers, uint32_t* err,
                                int max_ctas, cudaStream_t stream) {
  if ((off & 3) || (n & 3)) return -1;
  int grid = 132 * 2;  // = pb_grad_reduce_grid(): sumsq_partial has one slot per block of the widest launch
  if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;  // leave SMs to the backward pass this runs under
  mc_grad_reduce_kernel<<<grid, 512, 0, stream>>>(mc_grads, off, n, scale, out, sumsq_partial, wait_flags, slot_base, expect, npeers,
                                                  err);
  PB_CHECK_LAUNCH();
  return 0;
}
