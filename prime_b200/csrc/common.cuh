// Shared device helpers for the prime_b200 sm_90a kernel library.
// Everything here is plain CUDA C++ / inline PTX: no torch headers, no CUTLASS,
// so a full rebuild is seconds and the .so has a C ABI loaded through ctypes.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define PB_EXPORT extern "C" __attribute__((visibility("default")))

#define PB_CHECK_LAUNCH()                            \
  do {                                               \
    cudaError_t _e = cudaGetLastError();             \
    if (_e != cudaSuccess) return (int)_e;           \
  } while (0)

namespace pb {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum for blockDim.x <= 1024; `red` is >= 32 floats of shared memory.
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();  // protect `red` reuse across consecutive calls
  if (lane == 0) red[w] = v;
  __syncthreads();
  float t = (lane < nw) ? red[lane] : 0.f;
  t = warp_sum(t);
  return t;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float t = (lane < nw) ? red[lane] : -INFINITY;
  t = warp_max(t);
  return t;
}

struct __align__(16) bf16x8 {
  __nv_bfloat162 v[4];
};

__device__ __forceinline__ void unpack8(const bf16x8& p, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ bf16x8 pack8(const float (&f)[8]) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}

// Streaming 16-byte global accessors (no L1 allocation: these tensors are touched once).
__device__ __forceinline__ bf16x8 ldg_stream(const bf16x8* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return *reinterpret_cast<bf16x8*>(&r);
}
__device__ __forceinline__ void stg_stream(bf16x8* p, const bf16x8& v) {
  const uint4& r = *reinterpret_cast<const uint4*>(&v);
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(r.x), "r"(r.y), "r"(r.z),
               "r"(r.w));
}
// one 16-byte store (plain `*dst = v` on the struct is split into four 32-bit stores by the compiler: 4x the instructions and,
// on peer pointers, 4x the NVLink write packets)
__device__ __forceinline__ void stg_v4(bf16x8* p, const bf16x8& v) {
  const uint4& r = *reinterpret_cast<const uint4*>(&v);
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(r.x), "r"(r.y), "r"(r.z), "r"(r.w) : "memory");
}
__device__ __forceinline__ float4 ldg_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
// Coherent (non-.nc) vector load: required for peer / symmetric-heap data that another GPU wrote.
__device__ __forceinline__ float4 ld_relaxed_sys_f4(const float4* p) {
  float4 r;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ld_relaxed_sys_u4(const uint4* p) {
  uint4 r;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_acquire_gpu_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_add_release_gpu_u32(uint32_t* p, uint32_t v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

}  // namespace pb
