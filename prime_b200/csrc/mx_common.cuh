// The OCP MX e4m3 quantisation rule, shared by the MXFP8 GEMM operands (gemm_mxfp8_sm90.cu) and the e4m3 KV cache
// (decode_sm90.cu): per block of 32 values one UE8M0 power-of-two scale, values rounded to nearest-even with saturation.
#pragma once
#include <cuda_fp8.h>

#include "common.cuh"

namespace pb {

// smallest power of two s with amax / s <= 448 (e4m3 max), as a biased UE8M0 exponent; and 1/s
__device__ __forceinline__ uint32_t ue8m0_for(float amax, float& inv_scale) {
  const uint32_t bits = __float_as_uint(amax * (1.0f / 448.0f));
  uint32_t e = (bits >> 23) & 0xFF;
  if (bits & 0x7FFFFF) e += 1;
  e = min(max(e, 1u), 254u);
  inv_scale = __uint_as_float((254u - e) << 23);
  return e;
}
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}

}  // namespace pb
