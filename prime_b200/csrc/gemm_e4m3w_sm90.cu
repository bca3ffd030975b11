// e4m3 weights for generation: a skinny-M GEMM that reads MXFP8 weights in place, and their exact dequantisation.
//
//   C[M, N] (bf16, row stride ldc) = x[M, K] (bf16) · W̃ᵀ,   W̃[n, k] = e4m3(q[n, k]) · 2^(e[n, k/32] - 127),   1 <= M <= 64
//
// q and the UE8M0 exponents e are exactly what pb_quantize_mxfp8 writes (scale layout: gemm_mxfp8_sm90.cu). The tensor core sees
// bf16(W̃) and accumulates in fp32 on bf16 MMAs; activations are not quantised.
//
// A and B are swapped: weight rows sit on the M side of mma.m16n8k16 and tokens on its n = 8 side, so M = 1 pads to 8, not 128.
// A CTA of 4 warps owns 128 weight rows (32 per warp: two m16 tiles) and one K range of the split. It streams 128-byte K chunks
// through a 4-stage cp.async ring. Each thread copies exactly the weight bytes and exponents it will consume (its two rows of each
// tile, 32 contiguous bytes = one 32-block, and the 4-byte exponent word of the chunk), so those need no barrier; the x chunk is
// shared by the 4 warps and stored in fragment order, so every read of it is one conflict-free 16-byte load.
//
// K inside an MMA is permuted (A and B alike): lane t of a quad holds actual columns 32t + 4s .. 32t + 4s + 3 in MMA s of the chunk,
// so its 32 weight bytes of a row are contiguous and lie in one scale block.
//
// Dequantisation is exact and runs in registers: the e4m3 byte's magnitude shifted into bf16 position is e4m3 · 2^-120 (normals and
// subnormals alike), and one bf16 multiply by 2^(e - 7) gives W̃, rounded once (exact whenever W̃ is a bf16 normal). Blocks with
// e > 134, whose factor is above bf16's range, multiply twice (2^127, then 2^(e - 134)), the first exactly.
//
// Split-K (pb_gemm_e4m3w_splits) is a function of (M, N, K, SM count) only. With splits > 1 every CTA writes its fp32 partial of all
// its (m < M, n < N) into ws[split][M][N] and a second kernel sums the splits in index order: no atomics, so calls are deterministic.
#include <algorithm>

#include "common.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int kWarps = 4, kThreads = kWarps * 32;
constexpr int kTiles = 2;                         // m16 tiles (of weight rows) per warp
constexpr int kRows = kWarps * kTiles * 16;       // weight rows per CTA
constexpr int kChunk = 128;                       // K elements (= weight bytes) per stage
constexpr int kStages = 4;
constexpr int kWBytes = kThreads * kTiles * 64;   // per stage: each thread's 2 rows x 32 bytes per tile
constexpr int kSBytes = kThreads * kTiles * 8;    // per stage: each thread's 2 exponent words per tile
constexpr int M_MAX = 64;

template <int NG>  // token groups of 8: M <= 8·NG
__host__ __device__ constexpr int stage_bytes() { return kWBytes + kSBytes + NG * 2048; }

__device__ __forceinline__ size_t sf_word(int r, int chunk, int atoms) {
  // the 4 exponents of row r in K chunk `chunk` (blocks 4·chunk .. 4·chunk + 3) are one aligned word of the atom layout
  return ((size_t)chunk * atoms + (r >> 7)) * 512 + (size_t)((r & 31) * 16 + ((r & 127) >> 5) * 4);
}

__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}

__device__ __forceinline__ uint32_t bf16x2_mul(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}

// bytes (b0, b1) at selector positions of w → bf16x2 of e4m3 · 2^-120: each byte's sign to bit 15, its 7 magnitude bits to 4 .. 10
__device__ __forceinline__ uint32_t e4m3x2_bits(uint32_t w, uint32_t sel) {
  const uint32_t t = __byte_perm(w, 0, sel);  // byte b0 → bits 8..15, b1 → bits 24..31
  return (t & 0x80008000u) | ((t >> 4) & 0x07F007F0u);
}

struct E4m3wParams {
  int M, N, K, ldc, atoms, chunks_per_split, splits;
};

template <int NG>
__global__ void __launch_bounds__(kThreads, 1) gemm_e4m3w_kernel(const __nv_bfloat16* __restrict__ x, const uint8_t* __restrict__ q,
                                                              const uint8_t* __restrict__ sf, __nv_bfloat16* __restrict__ C,
                                                              float* __restrict__ ws, const E4m3wParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int kStage = stage_bytes<NG>();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n0 = (int)blockIdx.x * kRows + warp * (kTiles * 16);
  const int split = (int)blockIdx.y;
  const int c_begin = split * p.chunks_per_split;
  const int c_end = min(c_begin + p.chunks_per_split, p.K / kChunk);
  const int nchunks = c_end - c_begin;
  // this thread's weight rows (clamped: rows past N only feed accumulator rows that are never stored)
  const uint8_t* wrow[kTiles][2];
  int srow[kTiles][2];
#pragma unroll
  for (int i = 0; i < kTiles; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = min(n0 + i * 16 + g + h * 8, p.N - 1);
      wrow[i][h] = q + (int64_t)r * p.K + 32 * t;
      srow[i][h] = r;
    }
  // one stage: [weights: tile][half][16-byte piece][thread] | [exponent words: tile][half][thread] | [x: group][pair][lane]
  auto load = [&](int c, int st) {
    const uint32_t base = smem_u32(smem + st * kStage);
    const int kc = c_begin + c;
#pragma unroll
    for (int i = 0; i < kTiles; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint8_t* src = wrow[i][h] + (int64_t)kc * kChunk;
        cp_async16(base + (((i * 2 + h) * 2 + 0) * kThreads + threadIdx.x) * 16, src);
        cp_async16(base + (((i * 2 + h) * 2 + 1) * kThreads + threadIdx.x) * 16, src + 16);
        cp_async4(base + kWBytes + ((i * 2 + h) * kThreads + threadIdx.x) * 4, sf + sf_word(srow[i][h], kc, p.atoms));
      }
    // x: lane (g, t) of group j, pair u holds x[8j + g][128·kc + 32t + 8u .. + 7] (tokens past M clamped)
    for (int e = threadIdx.x; e < NG * 128; e += kThreads) {
      const int j = e >> 7, u = (e >> 5) & 3, l = e & 31;
      const int m = min(8 * j + (l >> 2), p.M - 1);
      cp_async16(base + kWBytes + kSBytes + e * 16, x + (int64_t)m * p.K + kc * kChunk + 32 * (l & 3) + 8 * u);
    }
  };
  float acc[kTiles][NG][4];
#pragma unroll
  for (int i = 0; i < kTiles; ++i)
#pragma unroll
    for (int j = 0; j < NG; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (s < nchunks) load(s, s);
    cp_async_commit();
  }
  for (int c = 0; c < nchunks; ++c) {
    cp_async_wait<kStages - 2>();
    __syncthreads();  // chunk c's x is visible to every warp, and the stage refilled below has been read by all
    if (c + kStages - 1 < nchunks) load(c + kStages - 1, (c + kStages - 1) % kStages);
    cp_async_commit();
    const uint8_t* base = smem + (c % kStages) * kStage;
    uint4 wv[kTiles][2][2];
    uint32_t s1[kTiles][2], s2[kTiles][2];
    bool big = false;
#pragma unroll
    for (int i = 0; i < kTiles; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        wv[i][h][0] = reinterpret_cast<const uint4*>(base)[((i * 2 + h) * 2 + 0) * kThreads + threadIdx.x];
        wv[i][h][1] = reinterpret_cast<const uint4*>(base)[((i * 2 + h) * 2 + 1) * kThreads + threadIdx.x];
        const uint32_t ew = reinterpret_cast<const uint32_t*>(base + kWBytes)[(i * 2 + h) * kThreads + threadIdx.x];
        const uint32_t e = (ew >> (8 * t)) & 0xFF;
        const uint32_t b1 = (min(e, 134u) + 120u) << 7, b2 = (max(e, 134u) - 7u) << 7;  // 2^(min(e,134)-7), 2^(max(e,134)-134)
        s1[i][h] = b1 | (b1 << 16);
        s2[i][h] = b2 | (b2 << 16);
        big |= e > 134u;
      }
    const uint4* xs = reinterpret_cast<const uint4*>(base + kWBytes + kSBytes);
#pragma unroll
    for (int u = 0; u < 4; ++u) {  // MMAs s = 2u, 2u + 1
      uint4 xv[NG];
#pragma unroll
      for (int j = 0; j < NG; ++j) xv[j] = xs[(j * 4 + u) * 32 + lane];
#pragma unroll
      for (int i = 0; i < kTiles; ++i) {
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          const int s = 2 * u + v;
          uint32_t a[4];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint4 w4 = wv[i][h][s >> 2];
            const uint32_t w = (s & 3) == 0 ? w4.x : (s & 3) == 1 ? w4.y : (s & 3) == 2 ? w4.z : w4.w;
            uint32_t lo = bf16x2_mul(e4m3x2_bits(w, 0x1404), s1[i][h]);  // columns 32t + 4s, +1
            uint32_t hi = bf16x2_mul(e4m3x2_bits(w, 0x3424), s1[i][h]);  // columns 32t + 4s + 2, +3
            if (big) {
              lo = bf16x2_mul(lo, s2[i][h]);
              hi = bf16x2_mul(hi, s2[i][h]);
            }
            a[h] = lo;      // a0a1 (row g) / a2a3 (row g + 8): logical k 2t, 2t+1
            a[2 + h] = hi;  // a4a5 / a6a7: logical k 2t+8, 2t+9
          }
#pragma unroll
          for (int j = 0; j < NG; ++j)
            mma16816(acc[i][j], a, v ? xv[j].z : xv[j].x, v ? xv[j].w : xv[j].y);
        }
      }
    }
  }
  cp_async_wait<0>();
  // acc[i][j]: c0 = (row g, token 2t), c1 = (row g, token 2t + 1), c2 / c3 = row g + 8
#pragma unroll
  for (int i = 0; i < kTiles; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = n0 + i * 16 + g + h * 8;
      if (n >= p.N) continue;
#pragma unroll
      for (int j = 0; j < NG; ++j)
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          const int m = 8 * j + 2 * t + v;
          if (m >= p.M) continue;
          const float val = acc[i][j][2 * h + v];
          if (p.splits == 1)
            C[(int64_t)m * p.ldc + n] = __float2bfloat16_rn(val);
          else
            ws[((int64_t)split * p.M + m) * p.N + n] = val;
        }
    }
}

// C[m, n] = bf16(Σ_s ws[s][m][n]), the splits summed in index order
__global__ void __launch_bounds__(256) e4m3w_reduce_kernel(const float* __restrict__ ws, __nv_bfloat16* __restrict__ C, int M, int N,
                                                           int ldc, int splits) {
  const int64_t total = (int64_t)M * N;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += ws[(int64_t)k * total + i];
    C[(i / N) * ldc + i % N] = __float2bfloat16_rn(s);
  }
}

// out[n, k] = bf16(W̃[n, k]): the e4m3 value exactly in fp32 (the bf16 bits times 2^120), times 2^(e - 127) exactly in fp32, rounded
// once to bf16, as the reference rounds its fp32 dequantisation. One thread per 32-block.
__global__ void __launch_bounds__(256) dequantize_mxfp8_kernel(const uint8_t* __restrict__ q, const uint8_t* __restrict__ sf,
                                                               __nv_bfloat16* __restrict__ out, int64_t ldo, int N, int K, int atoms) {
  const int bpr = K >> 5;
  const int64_t total = (int64_t)N * bpr;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / bpr), kb = (int)(i % bpr);
    const uint4* src = reinterpret_cast<const uint4*>(q + (int64_t)r * K + kb * 32);
    const uint32_t e = sf[sf_word(r, kb >> 2, atoms) + (kb & 3)];
    const float scale = __uint_as_float(e << 23);  // 2^(e - 127), a normal fp32 for every e in [1, 254]
    const uint4 v[2] = {src[0], src[1]};
    const uint32_t* w = reinterpret_cast<const uint32_t*>(v);
    uint32_t o[16];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const uint32_t b = e4m3x2_bits(w[j], hf ? 0x3424 : 0x1404);
        const float f0 = __uint_as_float(b << 16) * 0x1p120f, f1 = __uint_as_float(b & 0xFFFF0000u) * 0x1p120f;
        o[2 * j + hf] = pack_bf16(f0 * scale, f1 * scale);
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(out + (int64_t)r * ldo + kb * 32);
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[j] = make_uint4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
  }
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

template <int NG>
int launch_e4m3w(const void* x, const void* q, const void* sf, void* C, float* ws, const E4m3wParams& p, cudaStream_t stream) {
  static bool configured = false;
  constexpr int smem = kStages * stage_bytes<NG>();
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(gemm_e4m3w_kernel<NG>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const dim3 grid((p.N + kRows - 1) / kRows, p.splits);
  gemm_e4m3w_kernel<NG><<<grid, kThreads, smem, stream>>>((const __nv_bfloat16*)x, (const uint8_t*)q, (const uint8_t*)sf,
                                                          (__nv_bfloat16*)C, ws, p);
  return 0;
}

}  // namespace

// The largest M the skinny kernel takes; above it ops._matmul dequantises and runs the bf16 GEMM.
PB_EXPORT int pb_gemm_e4m3w_m_max() { return M_MAX; }

// Split-K count of pb_gemm_e4m3w: 1 when the row blocks alone fill the resident CTA slots of `num_sms` SMs (per SM as the stage
// size allows, at most 2); otherwise the fewest splits whose waves take the fewest chunk steps, with the fp32 partials (written and
// read once) capped at the weight bytes: s <= K / (8 · padded M).
PB_EXPORT int pb_gemm_e4m3w_splits(int M, int N, int K, int num_sms) {
  if (M < 1 || M > M_MAX || N < 1 || K < kChunk || K % kChunk != 0 || num_sms < 1) return -3;
  const int mp = M <= 8 ? 8 : M <= 16 ? 16 : M <= 32 ? 32 : 64;
  const int per_sm = std::max(1, (227 * 1024) / (kStages * (kWBytes + kSBytes + (mp / 8) * 2048)));
  const int slots = num_sms * std::min(per_sm, 2);
  const int blocks = (N + kRows - 1) / kRows, chunks = K / kChunk;
  if (blocks >= slots) return 1;
  const int cap = std::max(1, std::min(chunks, K / (8 * mp)));
  int best = 1;
  int64_t best_cost = INT64_MAX;
  for (int s = 1; s <= cap; ++s) {
    const int cps = (chunks + s - 1) / s;
    if (s > 1 && (chunks + cps - 1) / cps != s) continue;  // no empty split
    const int64_t cost = (int64_t)((blocks * s + slots - 1) / slots) * cps;
    if (cost < best_cost) best_cost = cost, best = s;
  }
  return best;
}

// C[M, N] (row stride ldc) = x[M, K] · W̃ᵀ. ws: fp32 [splits, M, N] when splits > 1 (else unused, may be null).
PB_EXPORT int pb_gemm_e4m3w(const void* x, const void* q, const void* sf, void* C, void* ws, int M, int N, int K, int ldc, int splits,
                            cudaStream_t stream) {
  if (x == nullptr || q == nullptr || sf == nullptr || C == nullptr || (splits > 1 && ws == nullptr)) return -1;
  if (K < kChunk || K % kChunk != 0) return -2;
  if (M < 1 || M > M_MAX || N < 1 || ldc < N) return -3;
  if (splits < 1 || splits > K / kChunk) return -5;
  if (!aligned(x, 16) || !aligned(q, 16) || !aligned(sf, 4) || !aligned(C, 2) || !aligned(ws, 4)) return -6;
  const int chunks = K / kChunk, cps = (chunks + splits - 1) / splits;
  if ((chunks + cps - 1) / cps != splits) return -5;  // an empty split would leave its partial unwritten
  const E4m3wParams p{M, N, K, ldc, (N + 127) / 128 + 1, cps, splits};
  float* w = splits > 1 ? (float*)ws : nullptr;
  const int ng = (M + 7) / 8;
  const int rc = ng == 1 ? launch_e4m3w<1>(x, q, sf, C, w, p, stream)
               : ng == 2 ? launch_e4m3w<2>(x, q, sf, C, w, p, stream)
               : ng <= 4 ? launch_e4m3w<4>(x, q, sf, C, w, p, stream)
                         : launch_e4m3w<8>(x, q, sf, C, w, p, stream);
  if (rc != 0) return rc;
  if (splits > 1) {
    const int64_t total = (int64_t)M * N;
    const int grid = (int)std::min<int64_t>((total + 255) / 256, 132 * 8);
    e4m3w_reduce_kernel<<<grid, 256, 0, stream>>>(w, (__nv_bfloat16*)C, M, N, ldc, splits);
  }
  PB_CHECK_LAUNCH();
  return 0;
}

// out[N, K] (row stride ldo) = bf16(W̃), bitwise equal to reference.dequantize_mxfp8(q, sf).to(bf16).
PB_EXPORT int pb_dequantize_mxfp8(const void* q, const void* sf, void* out, int N, int K, int64_t ldo, cudaStream_t stream) {
  if (q == nullptr || sf == nullptr || out == nullptr) return -1;
  if (K < kChunk || K % kChunk != 0) return -2;
  if (N < 1 || ldo < K) return -3;
  if (!aligned(q, 16) || !aligned(out, 16) || ldo % 8 != 0) return -6;
  const int64_t total = (int64_t)N * (K / 32);
  const int grid = (int)std::min<int64_t>((total + 255) / 256, 132 * 16);
  dequantize_mxfp8_kernel<<<grid, 256, 0, stream>>>((const uint8_t*)q, (const uint8_t*)sf, (__nv_bfloat16*)out, ldo, N, K, (N + 127) / 128 + 1);
  PB_CHECK_LAUNCH();
  return 0;
}
