// Block-scaled fp8 (MXFP8: e4m3 values, one UE8M0 power-of-two scale per 32 elements along K) GEMM for sm_90a, plus the
// quantisation kernels that produce its operands.
//
//   C[M,N] (bf16) = Σ_k  (A_q[m,k] · 2^(sfa[m,k/32]-127)) · (B_q[n,k] · 2^(sfb[n,k/32]-127))      fp32 accumulation
//
// Hopper's tensor core has no block-scaled MMA: every 32-element K block is one e4m3 mma.sync.m16n8k32 into a temporary fragment
// that is scaled by sfa[row]·sfb[col] and added to the fp32 accumulator in registers. (wgmma.m64nNk32 with e4m3 operands also
// covers exactly one scale block per instruction and would be the faster base for the same scheme; see DESIGN.md §1.6.)
//
// Scale-factor memory layout: for a [R, K] operand the buffer is  [K/128][ceil(R/128)+1][512 bytes]; one 512-byte "atom" covers
// 128 rows x 4 K-blocks and stores the byte of (row r, block kb) at  (r % 32) * 16 + ((r % 128) / 32) * 4 + kb.
//
// Tile 128 x 64 x 128 (K bytes), 4 warps of 32 x 64, operands staged in padded shared memory with cp.async (double-buffered).
#include <algorithm>

#include "common.cuh"
#include "mx_common.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int BM = 128, BN = 64, BKB = 128;  // BKB: K elements (= bytes) per stage
constexpr int kThreads = 128;
constexpr int kLd = BKB + 16;  // padded smem row (bytes): conflict-free ldmatrix
constexpr uint32_t kStageBytes = (BM + BN) * kLd + (BM + BN) * 4 * 4;  // A | B | scales [rows][4 blocks] fp32
constexpr uint32_t kSmemBytes = 2 * kStageBytes;

struct MxParams {
  int M, N, K;
  int atoms_m, atoms_n;
};

__device__ __forceinline__ size_t sf_offset(int r, int kblk, int atoms_r) {
  // kblk = index of the 32-element block along K
  return ((size_t)(kblk >> 2) * atoms_r + (r >> 7)) * 512 + (size_t)((r & 31) * 16 + ((r & 127) >> 5) * 4 + (kblk & 3));
}

__device__ __forceinline__ void mma_e4m3(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(kThreads) gemm_mxfp8_kernel(const uint8_t* __restrict__ A, const uint8_t* __restrict__ sfa,
                                                              const uint8_t* __restrict__ B, const uint8_t* __restrict__ sfb,
                                                              __nv_bfloat16* __restrict__ C, int ldc, const MxParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int m0 = (int)blockIdx.y * BM, n0 = (int)blockIdx.x * BN;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int ktiles = p.K / BKB;
  // rows past M / N are clamped to the last row: they only feed accumulator rows / columns that are never stored
  auto load = [&](int kt, int st) {
    uint8_t* base = smem + st * kStageBytes;
    const uint32_t sbase = smem_u32(base);
    for (int i = threadIdx.x; i < (BM + BN) * (BKB / 16); i += kThreads) {
      const int r = i / (BKB / 16), c = i % (BKB / 16);
      const uint8_t* src = r < BM ? A + (int64_t)min(m0 + r, p.M - 1) * p.K : B + (int64_t)min(n0 + r - BM, p.N - 1) * p.K;
      cp_async16(sbase + r * kLd + c * 16, src + kt * BKB + c * 16);
    }
    cp_async_commit();
    float* sc = reinterpret_cast<float*>(base + (BM + BN) * kLd);
    for (int i = threadIdx.x; i < (BM + BN) * 4; i += kThreads) {
      const int r = i >> 2, kb = kt * 4 + (i & 3);
      const uint32_t e = r < BM ? sfa[sf_offset(min(m0 + r, p.M - 1), kb, p.atoms_m)] : sfb[sf_offset(min(n0 + r - BM, p.N - 1), kb, p.atoms_n)];
      sc[i] = __uint_as_float(e << 23);
    }
  };
  float acc[2][8][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int n = 0; n < 8; ++n) acc[mi][n][0] = acc[mi][n][1] = acc[mi][n][2] = acc[mi][n][3] = 0.f;
  load(0, 0);
  for (int kt = 0; kt < ktiles; ++kt) {
    const int st = kt & 1;
    if (kt + 1 < ktiles) {
      load(kt + 1, st ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const uint8_t* base = smem + st * kStageBytes;
    const uint32_t sa = smem_u32(base), sb = sa + BM * kLd;
    const float* sc = reinterpret_cast<const float*>(base + (BM + BN) * kLd);
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {  // one UE8M0 block per k32 step
      uint32_t af[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
        ldsm_x4(sa + (warp * 32 + mi * 16 + (lane & 15)) * kLd + kb * 32 + (lane >> 4) * 16, af[mi]);
      float tmp[2][8][4];
#pragma unroll
      for (int n = 0; n < 8; n += 2) {
        uint32_t bf[4];
        ldsm_x4(sb + (n * 8 + (lane & 7) + (lane >> 4) * 8) * kLd + kb * 32 + ((lane >> 3) & 1) * 16, bf);
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          tmp[mi][n][0] = tmp[mi][n][1] = tmp[mi][n][2] = tmp[mi][n][3] = 0.f;
          tmp[mi][n + 1][0] = tmp[mi][n + 1][1] = tmp[mi][n + 1][2] = tmp[mi][n + 1][3] = 0.f;
          mma_e4m3(tmp[mi][n], af[mi], bf[0], bf[1]);
          mma_e4m3(tmp[mi][n + 1], af[mi], bf[2], bf[3]);
        }
      }
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const float s0 = sc[(warp * 32 + mi * 16 + g) * 4 + kb], s1 = sc[(warp * 32 + mi * 16 + g + 8) * 4 + kb];
#pragma unroll
        for (int n = 0; n < 8; ++n) {
          const float b0 = sc[(BM + n * 8 + 2 * t) * 4 + kb], b1 = sc[(BM + n * 8 + 2 * t + 1) * 4 + kb];
          acc[mi][n][0] = fmaf(tmp[mi][n][0], s0 * b0, acc[mi][n][0]);
          acc[mi][n][1] = fmaf(tmp[mi][n][1], s0 * b1, acc[mi][n][1]);
          acc[mi][n][2] = fmaf(tmp[mi][n][2], s1 * b0, acc[mi][n][2]);
          acc[mi][n][3] = fmaf(tmp[mi][n][3], s1 * b1, acc[mi][n][3]);
        }
      }
    }
    __syncthreads();  // this stage is refilled two iterations later
  }
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = m0 + warp * 32 + mi * 16 + g + h * 8;
      if (r >= p.M) continue;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const int c = n0 + n * 8 + 2 * t;
        if (c >= p.N) continue;  // N % 8 == 0
        const __nv_bfloat162 v = __floats2bfloat162_rn(acc[mi][n][2 * h], acc[mi][n][2 * h + 1]);
        *reinterpret_cast<__nv_bfloat162*>(C + (int64_t)r * ldc + c) = v;
      }
    }
}

// ---------------------------------------------------------------------------------------------------------------- quantisers
using pb::pack_e4m3x4;  // the MX rule (mx_common.cuh), shared with the e4m3 KV cache
using pb::ue8m0_for;

// x bf16 [R, C] (row stride ld) → q e4m3 [R, C] (dense) + scales for blocks of 32 along C. One thread per 32-element block.
__global__ void __launch_bounds__(256) quantize_mxfp8_kernel(const __nv_bfloat16* __restrict__ x, int64_t ld, uint8_t* __restrict__ q,
                                                             uint8_t* __restrict__ sf, int R, int C, int atoms_r) {
  const int blocks_per_row = C >> 5;
  const int64_t total = (int64_t)R * blocks_per_row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / blocks_per_row), kblk = (int)(i % blocks_per_row);
    const pb::bf16x8* src = reinterpret_cast<const pb::bf16x8*>(x + (int64_t)r * ld + kblk * 32);
    float f[32];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const pb::bf16x8 v = pb::ldg_stream(src + j);
      float t[8];
      pb::unpack8(v, t);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[j * 8 + e] = t[e];
    }
    float amax = 0.f;
#pragma unroll
    for (int e = 0; e < 32; ++e) amax = fmaxf(amax, fabsf(f[e]));
    float inv;
    const uint32_t e8 = ue8m0_for(amax, inv);
    uint4 o[2];
    uint32_t* ow = reinterpret_cast<uint32_t*>(o);
#pragma unroll
    for (int j = 0; j < 8; ++j) ow[j] = pack_e4m3x4(f[4 * j] * inv, f[4 * j + 1] * inv, f[4 * j + 2] * inv, f[4 * j + 3] * inv);
    uint4* dst = reinterpret_cast<uint4*>(q + (int64_t)r * C + kblk * 32);
    dst[0] = o[0];
    dst[1] = o[1];
    sf[sf_offset(r, kblk, atoms_r)] = (uint8_t)e8;
  }
}

// x bf16 [R, C] → qᵀ e4m3 [C, R] with scales for blocks of 32 along R (the contraction dim of the transposed use).
// Block: 128 rows x 32 columns through shared memory; thread t owns column (t % 32), row block (t / 32).
__global__ void __launch_bounds__(128) quantize_mxfp8_t_kernel(const __nv_bfloat16* __restrict__ x, int64_t ld, uint8_t* __restrict__ q,
                                                               uint8_t* __restrict__ sf, int R, int C, int atoms_c) {
  __shared__ float tile[128][33];
  const int r0 = blockIdx.y * 128, c0 = blockIdx.x * 32;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int rr = w; rr < 128; rr += 4) {
    const int r = r0 + rr, c = c0 + lane;
    tile[rr][lane] = (r < R && c < C) ? __bfloat162float(x[(int64_t)r * ld + c]) : 0.f;
  }
  __syncthreads();
  const int c = c0 + lane;
  const int rb = r0 + w * 32;
  if (c >= C || rb >= R) return;
  float f[32];
  float amax = 0.f;
#pragma unroll
  for (int e = 0; e < 32; ++e) {
    f[e] = tile[w * 32 + e][lane];
    amax = fmaxf(amax, fabsf(f[e]));
  }
  float inv;
  const uint32_t e8 = ue8m0_for(amax, inv);
  uint4 o[2];
  uint32_t* ow = reinterpret_cast<uint32_t*>(o);
#pragma unroll
  for (int j = 0; j < 8; ++j) ow[j] = pack_e4m3x4(f[4 * j] * inv, f[4 * j + 1] * inv, f[4 * j + 2] * inv, f[4 * j + 3] * inv);
  uint4* dst = reinterpret_cast<uint4*>(q + (int64_t)c * R + rb);
  dst[0] = o[0];
  dst[1] = o[1];
  sf[sf_offset(c, rb >> 5, atoms_c)] = (uint8_t)e8;
}

}  // namespace

// transpose = 0: q [R, C] with blocks along C (C % 128 == 0).   transpose = 1: q [C, R] with blocks along R (R % 128 == 0).
PB_EXPORT int pb_quantize_mxfp8(const void* x, int64_t ld, void* q, void* sf, int R, int C, int transpose, cudaStream_t stream) {
  if (R <= 0 || C <= 0) return 0;
  if ((ld % 8) || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q)) & 15)) return -1;
  if (!transpose) {
    if (C % 128) return -2;
    const int64_t total = (int64_t)R * (C / 32);
    const int grid = (int)std::min<int64_t>((total + 255) / 256, 132 * 16);
    quantize_mxfp8_kernel<<<grid, 256, 0, stream>>>((const __nv_bfloat16*)x, ld, (uint8_t*)q, (uint8_t*)sf, R, C, (R + 127) / 128 + 1);
  } else {
    if (R % 128) return -2;
    dim3 grid((C + 31) / 32, R / 128);
    quantize_mxfp8_t_kernel<<<grid, 128, 0, stream>>>((const __nv_bfloat16*)x, ld, (uint8_t*)q, (uint8_t*)sf, R, C, (C + 127) / 128 + 1);
  }
  PB_CHECK_LAUNCH();
  return 0;
}

// C[M,N] bf16 = A_q[M,K] · B_q[N,K]ᵀ with per-32 UE8M0 scales (buffers laid out as described at the top of this file).
PB_EXPORT int pb_gemm_mxfp8(const void* Aq, const void* sfa, const void* Bq, const void* sfb, void* C, int M, int N, int K, int ldc,
                            cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (K % 128 || ldc % 8 || N % 8) return -1;
  if ((reinterpret_cast<uintptr_t>(Aq) | reinterpret_cast<uintptr_t>(Bq) | reinterpret_cast<uintptr_t>(C)) & 15) return -2;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_mxfp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  MxParams p{M, N, K, (M + 127) / 128 + 1, (N + 127) / 128 + 1};
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  gemm_mxfp8_kernel<<<grid, kThreads, kSmemBytes, stream>>>((const uint8_t*)Aq, (const uint8_t*)sfa, (const uint8_t*)Bq, (const uint8_t*)sfb,
                                                            (__nv_bfloat16*)C, ldc, p);
  PB_CHECK_LAUNCH();
  return 0;
}
