// Token-by-token generation over a KV cache: the per-step bookkeeping, the append of the new token's rotated K / V, and split-KV
// ("flash-decoding") attention of one query per sequence over a long cache.
//
// Cache layout, per layer: kv [B, capacity, 2·Hkv·D] bf16 = exactly the K | V columns of the fused QKV row, K already rotated. K head
// hk sits at column hk·D, V head hk at column (Hkv + hk)·D. Per-row device state (int32 [B] len / lo, int64 [B] last_tok) lives on
// the device, so a decode step needs no host value that changes between tokens and can be replayed from a CUDA graph.
//
// Visibility is the rule of pb_doc_bounds and the training kernels: the query of row b (at position len[b] - 1) sees key k iff
// max(lo[b], len[b] - window) <= k < len[b] (window 0 = none, lo null = 0).
//
// A verify step (speculative decoding) runs T tokens per row at once: query t of row b sits at position len[b] - T + t and sees key
// k iff max(lo[b, t], pos + 1 - window) <= k <= pos, with lo [B, T] the document start of each query.
//
// An e4m3 cache (the *_fp8 launchers) has the same layout in bytes, kv uint8 [B, capacity, 2·Hkv·D], plus kv_scale uint8
// [B, capacity, 2·Hkv·D/32]: byte j of a row is the UE8M0 exponent e of its columns 32j .. 32j+31 (scale 2^(e-127)). The values are
// the MX quantisation (mx_common.cuh) of exactly what the bf16 cache would hold: K after its one bf16 rounding, V as is. Every
// dequantised value is exact in fp32, so attention over the e4m3 cache is attention over a known bf16 cache.
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "mx_common.cuh"

namespace {

using pb::bf16x8;

// -------------------------------------------------------------------------------------------------------------- step bookkeeping
__global__ void decode_advance_kernel(const int64_t* __restrict__ tokens, int64_t eos, int* __restrict__ len, int* __restrict__ lo,
                                      int64_t* __restrict__ last_tok, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int pos = len[b];
  if (last_tok[b] == eos) lo[b] = pos;  // the previous token ended a document: this one starts the next (eos < 0 never matches)
  len[b] = pos + 1;
  last_tok[b] = tokens[b];
}

// T tokens per row in one step: the same rule applied token after token, with each query's document start written to lo_q [B, T]
__global__ void verify_advance_kernel(const int64_t* __restrict__ tokens, int T, int64_t eos, int* __restrict__ len, int* __restrict__ lo,
                                      int* __restrict__ lo_q, int64_t* __restrict__ last_tok, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int pos = len[b];
  int l = lo[b];
  int64_t last = last_tok[b];
  for (int t = 0; t < T; ++t) {
    if (last == eos) l = pos + t;
    lo_q[(int64_t)b * T + t] = l;
    last = tokens[(int64_t)b * T + t];
  }
  len[b] = pos + T;
  lo[b] = l;
  last_tok[b] = last;
}

// ------------------------------------------------------------------------------------------------------------------ KV append
// Columns 8·vh .. 8·vh+7 of a Q or K head rotated at position pos: interleaved pairs, fp32, one bf16 rounding.
__device__ __forceinline__ bf16x8 rope8(const bf16x8& x, const float4* __restrict__ cosb, const float4* __restrict__ sinb, int pos, int vec,
                                       int vh) {
  float v[8], o[8];
  pb::unpack8(x, v);
  const float4 c = cosb[(int64_t)pos * vec + vh], s = sinb[(int64_t)pos * vec + vh];
  const float cc[4] = {c.x, c.y, c.z, c.w}, sn[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    o[2 * j] = v[2 * j] * cc[j] - v[2 * j + 1] * sn[j];
    o[2 * j + 1] = v[2 * j] * sn[j] + v[2 * j + 1] * cc[j];
  }
  return pb::pack8(o);
}

// One token's fused row at position pos: Q heads are rotated in place, K heads are rotated into the cache row dst, V heads are
// copied; the rotation is rope_inplace_kernel's (interleaved pairs, fp32, one bf16 rounding).
__device__ __forceinline__ void append_row(bf16x8* __restrict__ row, bf16x8* __restrict__ dst, const float4* __restrict__ cosb,
                                           const float4* __restrict__ sinb, int pos, int H, int Hkv, int vec) {
  const int n = (H + 2 * Hkv) * vec;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int head = i / vec, vh = i - head * vec;
    bf16x8 x = row[i];
    if (head < H + Hkv) x = rope8(x, cosb, sinb, pos, vec, vh);
    if (head < H)
      row[i] = x;
    else
      dst[i - H * vec] = x;
  }
}

// One CTA per row. Position pos = len[b] - 1 (rows outside [0, capacity) are left alone).
__global__ void __launch_bounds__(128) kv_append_kernel(bf16x8* __restrict__ qkv, bf16x8* __restrict__ kv, const int* __restrict__ len,
                                                        const float4* __restrict__ cosb, const float4* __restrict__ sinb, int H, int Hkv,
                                                        int vec, int capacity) {
  const int b = blockIdx.x;
  const int pos = len[b] - 1;
  if (pos < 0 || pos >= capacity) return;
  const int n = (H + 2 * Hkv) * vec;
  append_row(qkv + (int64_t)b * n, kv + ((int64_t)b * capacity + pos) * (2 * Hkv * vec), cosb, sinb, pos, H, Hkv, vec);
}

// One CTA per (token, row): token t of row b at position len[b] - T + t.
__global__ void __launch_bounds__(128) kv_append_tokens_kernel(bf16x8* __restrict__ qkv, bf16x8* __restrict__ kv, const int* __restrict__ len,
                                                               const float4* __restrict__ cosb, const float4* __restrict__ sinb, int T, int H,
                                                               int Hkv, int vec, int capacity) {
  const int t = blockIdx.x, b = blockIdx.y;
  const int pos = len[b] - T + t;
  if (pos < 0 || pos >= capacity) return;
  const int n = (H + 2 * Hkv) * vec;
  append_row(qkv + ((int64_t)b * T + t) * n, kv + ((int64_t)b * capacity + pos) * (2 * Hkv * vec), cosb, sinb, pos, H, Hkv, vec);
}

// ------------------------------------------------------------------------------------------------------------- e4m3 cache writes
// A thread holds 8 columns, so the 4 lanes of an aligned quad hold one 32-column block (D % 32 == 0: a block never straddles two
// heads). The quad's amax takes two shuffles; the lane holding the block's first columns writes its exponent.
__device__ __forceinline__ float quad_amax(const float (&f)[8]) {
  float a = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) a = fmaxf(a, fabsf(f[j]));
  a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 1));
  return fmaxf(a, __shfl_xor_sync(0xffffffffu, a, 2));
}

// Columns 8c .. 8c+7 of a cache row (f, already at their bf16 values) into e4m3 bytes dst[c] and, for c % 4 == 0, exponent sdst[c/4].
__device__ __forceinline__ void store_e4m3x8(const float (&f)[8], float amax, uint2* __restrict__ dst, uint8_t* __restrict__ sdst, int c) {
  float inv;
  const uint32_t e = pb::ue8m0_for(amax, inv);
  dst[c] = make_uint2(pb::pack_e4m3x4(f[0] * inv, f[1] * inv, f[2] * inv, f[3] * inv),
                      pb::pack_e4m3x4(f[4] * inv, f[5] * inv, f[6] * inv, f[7] * inv));
  if ((c & 3) == 0) sdst[c >> 2] = (uint8_t)e;
}

// kv_append_tokens_kernel into an e4m3 cache: one CTA per (token, row), token t of row b at position len[b] - T + t. Q heads are
// rotated in place as there; K heads are rotated and rounded to bf16, then quantised with V into the cache row.
__global__ void __launch_bounds__(128) kv_append_fp8_kernel(bf16x8* __restrict__ qkv, uint2* __restrict__ kv, uint8_t* __restrict__ kv_scale,
                                                            const int* __restrict__ len, const float4* __restrict__ cosb,
                                                            const float4* __restrict__ sinb, int T, int H, int Hkv, int vec, int capacity) {
  const int t = blockIdx.x, b = blockIdx.y;
  const int pos = len[b] - T + t;
  if (pos < 0 || pos >= capacity) return;
  const int n = (H + 2 * Hkv) * vec;
  bf16x8* row = qkv + ((int64_t)b * T + t) * n;
  const int64_t r = (int64_t)b * capacity + pos;
  uint2* dst = kv + r * (2 * Hkv * vec);
  uint8_t* sdst = kv_scale + r * (2 * Hkv * vec / 4);
  for (int i0 = 0; i0 < n; i0 += blockDim.x) {  // a bound uniform over the warp: the quad shuffles need every lane
    const int i = i0 + threadIdx.x;
    const int head = i / vec;
    bf16x8 x{};
    float f[8] = {};
    if (i < n) {
      x = row[i];
      if (head < H + Hkv) x = rope8(x, cosb, sinb, pos, vec, i - head * vec);
      pb::unpack8(x, f);
    }
    const float amax = quad_amax(f);  // n % 4 == 0: a quad is wholly inside or wholly past the row, and inside one head
    if (i >= n) continue;
    if (head < H)
      row[i] = x;
    else
      store_e4m3x8(f, amax, dst, sdst, i - H * vec);
  }
}

// Prefill: bf16 rows src + (b·S + s)·ld, cols wide, into e4m3 cache rows s = 0 .. S-1 of row b. One thread per 8 columns.
__global__ void __launch_bounds__(256) kv_quantize_kernel(const __nv_bfloat16* __restrict__ src, int64_t ld, uint2* __restrict__ kv,
                                                          uint8_t* __restrict__ kv_scale, int S, int vec, int capacity, int64_t total) {
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x; i0 < total; i0 += (int64_t)gridDim.x * blockDim.x) {  // uniform bound
    const int64_t i = i0 + threadIdx.x;
    const int64_t r = i / vec;  // b·S + s
    const int c = (int)(i - r * vec);
    float f[8] = {};
    if (i < total) pb::unpack8(pb::ldg_stream(reinterpret_cast<const bf16x8*>(src + r * ld + c * 8)), f);
    const float amax = quad_amax(f);
    if (i >= total) continue;
    const int64_t b = r / S, row = b * capacity + (r - b * S);
    store_e4m3x8(f, amax, kv + row * vec, kv_scale + row * (vec / 4), c);
  }
}

// ------------------------------------------------------------------------------------------------------------- split-KV attention
struct DecodeParams {
  const __nv_bfloat16* qkv;  // [B, (H + 2Hkv)·D], Q rotated ([B, T, ·] when verifying)
  const __nv_bfloat16* kv;   // [B, capacity, 2·Hkv·D]
  const int* len;
  const int* lo;  // nullable; [B, T] when verifying
  __nv_bfloat16* out;  // [B, H·D] ([B, T, H·D] when verifying)
  float* part;         // [B, H, splits, D + 2] ([B, T, H, ...]): unnormalised accumulator, running max (log2 domain), sum
  int H, Hkv, G, chunks, capacity, window, splits, keys_per_split;
  float scale_log2;
  int T;  // verify: tokens per row
  const uint8_t* kv_scale;  // e4m3 cache: [B, capacity, 2·Hkv·D/32] UE8M0 exponents (kv then holds the e4m3 bytes)
};

// 8 e4m3 values (one 8-byte load) → fp32, exactly: cvt.rn.f16x2.e4m3x2 per pair, the low byte the lower column
__device__ __forceinline__ void unpack8_e4m3(const uint2& x, float (&f)[8]) {
  const uint32_t w[2] = {x.x, x.y};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t h2;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"((unsigned short)(w[i >> 1] >> (16 * (i & 1)))));
    const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&h2));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint2 ldg_stream8(const uint8_t* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ float ue8m0_scale(uint8_t e) { return __uint_as_float((uint32_t)e << 23); }  // 2^(e-127), e in [1, 254]

constexpr int kDecThreads = 128;
constexpr int kDecWarps = kDecThreads / 32;

// Grid (split, kv head × query chunk, row). A CTA owns GC <= 8 query vectors of one GQA group, so every K / V byte of its key range
// is read once per chunk of 8 query vectors. Decoding, the vectors are the chunk's heads of the group (G <= 8: once per step);
// verifying (kMulti), they are the (token t, head g) pairs j = t·G + g of the T·G queries of the group, each with its own key range,
// and the CTA's key loop covers the union of those ranges. A lane group of D/8 lanes holds one key, each lane 8 of its dimensions; a
// warp covers 32·8/D keys per load and every lane keeps kUnroll keys' K and V loads in flight. Scores are reduced over the lane group
// by shuffles; each lane group runs its own online softmax, and the groups are merged (shuffles, then shared memory) at the end.
//
// kFp8: the cache holds e4m3 bytes with a UE8M0 exponent per 32 columns. A lane loads its 8 K and 8 V bytes (8-byte streaming
// loads) and its blocks' two exponents, converts exactly, and applies the power-of-two scales as products that round nothing: K's
// to its partial dot product before the lane-group reduction, V's to p before the V FMA. Every sum is then the bf16 kernel's sum
// over the dequantised cache.
template <int D, int GC, bool kMulti, bool kFp8 = false>
__device__ __forceinline__ void attn_body(const DecodeParams& p) {
  constexpr int LPK = D / 8;   // lanes per key
  constexpr int KPW = 32 / LPK;  // keys per warp and load
  constexpr int kUnroll = GC >= 8 ? 2 : 4;  // the fp8 kernels too: 8 keys per lane halved occupancy (DESIGN.md §1.5)
  constexpr int KPI = kDecWarps * KPW * kUnroll;  // keys per CTA iteration
  __shared__ float s_m[kDecWarps][GC], s_l[kDecWarps][GC];
  __shared__ float s_acc[kDecWarps][GC][D];

  const int split = blockIdx.x, b = blockIdx.z;
  const int hk = blockIdx.y / p.chunks, c = blockIdx.y - hk * p.chunks;
  const int h0 = hk * p.G + c * GC, ng = min(GC, (kMulti ? p.T * p.G : p.G) - c * GC);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, grp = lane / LPK, sub = lane % LPK;
  int qb[kMulti ? GC : 1], qe[kMulti ? GC : 1];  // verify: each query vector's keys [qb, qe)
  const int2 kr = [&]() {
    if constexpr (kMulti) {
      const int len = p.len[b];
      int ub = 0, lb = INT_MAX;
#pragma unroll
      for (int g = 0; g < GC; ++g) {
        const int t = (c * GC + g) / p.G;
        const int e = min(len - p.T + t + 1, p.capacity);
        int kb = p.lo != nullptr ? p.lo[(int64_t)b * p.T + min(t, p.T - 1)] : 0;
        if (p.window > 0) kb = max(kb, e - p.window);
        kb = max(kb, 0);
        qb[g] = g < ng ? kb : 0;
        qe[g] = g < ng ? e : 0;
        if (g < ng && kb < e) {
          lb = min(lb, kb);
          ub = max(ub, e);
        }
      }
      const int s0 = split * p.keys_per_split;
      return make_int2(max(lb, s0), min(ub, s0 + p.keys_per_split));
    } else {
      const int L = min(p.len[b], p.capacity);
      int kbeg = p.lo != nullptr ? p.lo[b] : 0;
      if (p.window > 0) kbeg = max(kbeg, L - p.window);
      const int s0 = split * p.keys_per_split;
      return make_int2(max(max(kbeg, 0), s0), min(L, s0 + p.keys_per_split));
    }
  }();
  const int k0 = kr.x, k1 = kr.y;

  const int ldq = (p.H + 2 * p.Hkv) * D, ldkv = 2 * p.Hkv * D;
  float m[GC], l[GC], acc[GC][8];
#pragma unroll
  for (int g = 0; g < GC; ++g) {
    m[g] = -INFINITY;
    l[g] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[g][j] = 0.f;
  }

  if (k0 < k1) {  // an empty key range (window, length or a split past the end) skips straight to writing an empty partial
    float q[GC][8];
#pragma unroll
    for (int g = 0; g < GC; ++g) {
      if (g < ng) {
        if constexpr (kMulti) {
          const int j = c * GC + g, t = j / p.G;
          const __nv_bfloat16* qp = p.qkv + ((int64_t)b * p.T + t) * ldq + (hk * p.G + j - t * p.G) * D;
          pb::unpack8(*reinterpret_cast<const bf16x8*>(qp + sub * 8), q[g]);
        } else {
          pb::unpack8(*reinterpret_cast<const bf16x8*>(p.qkv + (int64_t)b * ldq + (h0 + g) * D + sub * 8), q[g]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) q[g][j] *= p.scale_log2;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) q[g][j] = 0.f;
      }
    }
    const __nv_bfloat16* kbase = p.kv + (int64_t)b * p.capacity * ldkv + hk * D + sub * 8;
    const __nv_bfloat16* vbase = kbase + p.Hkv * D;
    // e4m3 cache: one byte per column, one exponent per 32 columns (the lane's 8 columns lie in one block)
    const uint8_t* kbase8 = reinterpret_cast<const uint8_t*>(p.kv) + (int64_t)b * p.capacity * ldkv + hk * D + sub * 8;
    const uint8_t* sbase = p.kv_scale + (int64_t)b * p.capacity * (ldkv / 32) + (hk * D + sub * 8) / 32;
    // the loop bound is uniform over the warp (the shuffles below need every lane); keys past k1 are loaded by no lane and score -inf
    for (int wb = k0 + warp * KPW * kUnroll; wb < k1; wb += KPI) {
      const int base = wb + grp;
      using Raw = std::conditional_t<kFp8, uint2, bf16x8>;
      Raw kr[kUnroll] = {}, vr[kUnroll] = {};
      uint8_t ke[kFp8 ? kUnroll : 1] = {}, ve[kFp8 ? kUnroll : 1] = {};
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int key = base + u * KPW;
        if (key < k1) {
          if constexpr (kFp8) {
            kr[u] = ldg_stream8(kbase8 + (int64_t)key * ldkv);
            vr[u] = ldg_stream8(kbase8 + (int64_t)key * ldkv + p.Hkv * D);
            ke[u] = __ldg(sbase + (int64_t)key * (ldkv / 32));
            ve[u] = __ldg(sbase + (int64_t)key * (ldkv / 32) + p.Hkv * D / 32);
          } else {
            kr[u] = pb::ldg_stream(reinterpret_cast<const bf16x8*>(kbase + (int64_t)key * ldkv));
            vr[u] = pb::ldg_stream(reinterpret_cast<const bf16x8*>(vbase + (int64_t)key * ldkv));
          }
        }
      }
      float s[kUnroll][GC];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        float kf[8];
        if constexpr (kFp8)
          unpack8_e4m3(kr[u], kf);
        else
          pb::unpack8(kr[u], kf);
#pragma unroll
        for (int g = 0; g < GC; ++g) {
          float d = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) d = fmaf(q[g][j], kf[j], d);
          if constexpr (kFp8) d *= ue8m0_scale(ke[u]);
#pragma unroll
          for (int o = LPK / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
          if constexpr (kMulti) {
            const int key = base + u * KPW;
            s[u][g] = key < k1 && key >= qb[g] && key < qe[g] ? d : -INFINITY;
          } else {
            s[u][g] = base + u * KPW < k1 ? d : -INFINITY;
          }
        }
      }
#pragma unroll
      for (int g = 0; g < GC; ++g) {
        float mx = m[g];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) mx = fmaxf(mx, s[u][g]);
        const float ms = mx == -INFINITY ? 0.f : mx;  // a lane group with no valid key yet: keep everything at zero, no NaN
        const float corr = exp2f(m[g] - ms);
        m[g] = mx;
        l[g] *= corr;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[g][j] *= corr;
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) s[u][g] = exp2f(s[u][g] - ms);
      }
      // a key outside one query's range but inside the union has weight 0 for it; every key below len is a written cache row
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        if (base + u * KPW >= k1) continue;
        float vf[8];
        if constexpr (kFp8)
          unpack8_e4m3(vr[u], vf);
        else
          pb::unpack8(vr[u], vf);
#pragma unroll
        for (int g = 0; g < GC; ++g) {
          l[g] += s[u][g];
          const float pv = kFp8 ? s[u][g] * ue8m0_scale(ve[u]) : s[u][g];
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[g][j] = fmaf(pv, vf[j], acc[g][j]);
        }
      }
    }
  }

  // merge the lane groups of the warp (same dimensions, different keys), then the warps through shared memory
#pragma unroll
  for (int o = LPK; o < 32; o <<= 1) {
#pragma unroll
    for (int g = 0; g < GC; ++g) {
      const float mo = __shfl_xor_sync(0xffffffffu, m[g], o), lo_ = __shfl_xor_sync(0xffffffffu, l[g], o);
      const float mx = fmaxf(m[g], mo), ms = mx == -INFINITY ? 0.f : mx;
      const float a = exp2f(m[g] - ms), bb = exp2f(mo - ms);
      m[g] = mx;
      l[g] = l[g] * a + lo_ * bb;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[g][j] = acc[g][j] * a + __shfl_xor_sync(0xffffffffu, acc[g][j], o) * bb;
    }
  }
  if (grp == 0) {
#pragma unroll
    for (int g = 0; g < GC; ++g) {
      if (sub == 0) {
        s_m[warp][g] = m[g];
        s_l[warp][g] = l[g];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s_acc[warp][g][sub * 8 + j] = acc[g][j];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < ng * D; i += kDecThreads) {
    const int g = i / D, d = i - g * D;
    float mx = -INFINITY;
#pragma unroll
    for (int w = 0; w < kDecWarps; ++w) mx = fmaxf(mx, s_m[w][g]);
    const float ms = mx == -INFINITY ? 0.f : mx;
    float sum = 0.f, a = 0.f;
#pragma unroll
    for (int w = 0; w < kDecWarps; ++w) {
      const float e = exp2f(s_m[w][g] - ms);
      sum += s_l[w][g] * e;
      a += s_acc[w][g][d] * e;
    }
    if constexpr (kMulti) {
      const int j = c * GC + g, t = j / p.G;
      const int64_t bh = ((int64_t)b * p.T + t) * p.H + hk * p.G + j - t * p.G;  // output row (b, t, h)
      if (p.splits == 1) {
        p.out[bh * D + d] = __float2bfloat16_rn(sum > 0.f ? a / sum : 0.f);
      } else {
        float* pp = p.part + (bh * p.splits + split) * (D + 2);
        pp[d] = a;
        if (d == 0) {
          pp[D] = mx;
          pp[D + 1] = sum;
        }
      }
      continue;
    }
    const int h = h0 + g;
    if (p.splits == 1) {
      p.out[(int64_t)b * p.H * D + h * D + d] = __float2bfloat16_rn(sum > 0.f ? a / sum : 0.f);
    } else {
      float* pp = p.part + (((int64_t)b * p.H + h) * p.splits + split) * (D + 2);
      pp[d] = a;
      if (d == 0) {
        pp[D] = mx;
        pp[D + 1] = sum;
      }
    }
  }
}

template <int D, int GC>
__global__ void __launch_bounds__(kDecThreads) decode_attn_kernel(const DecodeParams p) {
  attn_body<D, GC, false>(p);
}

template <int D, int GC>
__global__ void __launch_bounds__(kDecThreads) verify_attn_kernel(const DecodeParams p) {
  attn_body<D, GC, true>(p);
}

// Combine the partials of every split in split order (deterministic): one CTA per (row, head), one thread per dimension.
__global__ void __launch_bounds__(128) decode_combine_kernel(const float* __restrict__ part, __nv_bfloat16* __restrict__ out, int H, int D,
                                                             int splits) {
  const int bh = blockIdx.x;
  const float* pp = part + (int64_t)bh * splits * (D + 2);
  float mx = -INFINITY;
  for (int s = 0; s < splits; ++s) mx = fmaxf(mx, pp[s * (D + 2) + D]);
  const float ms = mx == -INFINITY ? 0.f : mx;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float sum = 0.f, a = 0.f;
    for (int s = 0; s < splits; ++s) {
      const float e = exp2f(pp[s * (D + 2) + D] - ms);
      sum += pp[s * (D + 2) + D + 1] * e;
      a += pp[s * (D + 2) + d] * e;
    }
    out[(int64_t)bh * D + d] = __float2bfloat16_rn(sum > 0.f ? a / sum : 0.f);
  }
}

template <int D, int GC>
__global__ void __launch_bounds__(kDecThreads) decode_attn_fp8_kernel(const DecodeParams p) {
  attn_body<D, GC, false, true>(p);
}

template <int D, int GC>
__global__ void __launch_bounds__(kDecThreads) verify_attn_fp8_kernel(const DecodeParams p) {
  attn_body<D, GC, true, true>(p);
}

template <int D, int GC, bool kMulti, bool kFp8>
void attn_kernel(dim3 grid, const DecodeParams& p, cudaStream_t stream) {
  if constexpr (kMulti && kFp8) verify_attn_fp8_kernel<D, GC><<<grid, kDecThreads, 0, stream>>>(p);
  else if constexpr (kMulti) verify_attn_kernel<D, GC><<<grid, kDecThreads, 0, stream>>>(p);
  else if constexpr (kFp8) decode_attn_fp8_kernel<D, GC><<<grid, kDecThreads, 0, stream>>>(p);
  else decode_attn_kernel<D, GC><<<grid, kDecThreads, 0, stream>>>(p);
}

// Decoding, the G query heads of a KV group; verifying (kMulti), its T·G query vectors: in chunks of the smallest power of two
// >= that count, at most 8 (more: several chunks of 8). Then the combine over the B·T·H output rows when the keys are split.
template <int D, bool kMulti, bool kFp8>
int launch_attn(const DecodeParams& p0, int B, cudaStream_t stream) {
  DecodeParams p = p0;
  const int nq = kMulti ? p.T * p.G : p.G;
  const int gc = nq > 4 ? 8 : nq > 2 ? 4 : nq;
  p.chunks = (nq + gc - 1) / gc;
  const dim3 grid(p.splits, p.Hkv * p.chunks, B);
  if (gc == 8) attn_kernel<D, 8, kMulti, kFp8>(grid, p, stream);
  else if (gc == 4) attn_kernel<D, 4, kMulti, kFp8>(grid, p, stream);
  else if (gc == 2) attn_kernel<D, 2, kMulti, kFp8>(grid, p, stream);
  else attn_kernel<D, 1, kMulti, kFp8>(grid, p, stream);
  if (p.splits > 1) decode_combine_kernel<<<B * p.T * p.H, 128, 0, stream>>>(p.part, p.out, p.H, D, p.splits);
  PB_CHECK_LAUNCH();
  return 0;
}

inline bool aligned(const void* ptr, uintptr_t a) { return ((uintptr_t)ptr & (a - 1)) == 0; }

constexpr int kSplitKeys = 64;  // a split covers a whole number of 64-key tiles of the capacity

}  // namespace

// Return codes of the decode launchers, checked before the first CUDA call: -1 a required pointer is null, -2 D is not 64 or 128,
// -3 an impossible shape (B, H, Hkv or capacity < 1, H % Hkv != 0), -4 window < 0, -5 splits < 1, -6 a misaligned pointer (16 bytes
// for bf16 / fp32 vectors, 4 for the int32 state and the fp32 workspace, 8 for int64).

// At the start of every decode step, per row: pos = len; lo = (last_tok == eos) ? pos : lo; len = pos + 1; last_tok = tokens.
// tokens int64 [B]; eos < 0 = no documents.
PB_EXPORT int pb_decode_advance(const int64_t* tokens, int64_t eos, int* len, int* lo, int64_t* last_tok, int B, cudaStream_t stream) {
  if (tokens == nullptr || len == nullptr || lo == nullptr || last_tok == nullptr) return -1;
  if (B < 1) return -3;
  if (!aligned(tokens, 8) || !aligned(last_tok, 8) || !aligned(len, 4) || !aligned(lo, 4)) return -6;
  decode_advance_kernel<<<(B + 127) / 128, 128, 0, stream>>>(tokens, eos, len, lo, last_tok, B);
  PB_CHECK_LAUNCH();
  return 0;
}

// qkv: the new token's un-rotated fused row, contiguous [B, (H + 2Hkv)·D] bf16; kv: the layer's cache [B, capacity, 2·Hkv·D];
// cos / sin: fp32 [>= capacity, D/2]. At position len[b] - 1: Q heads rotated in place, rotated K and V written to that cache row.
PB_EXPORT int pb_kv_append(void* qkv, void* kv, const int* len, const float* cos, const float* sin, int B, int H, int Hkv, int D,
                           int capacity, cudaStream_t stream) {
  if (qkv == nullptr || kv == nullptr || len == nullptr || cos == nullptr || sin == nullptr) return -1;
  if (D != 64 && D != 128) return -2;
  if (B < 1 || H < 1 || Hkv < 1 || capacity < 1 || H % Hkv != 0) return -3;
  if (!aligned(qkv, 16) || !aligned(kv, 16) || !aligned(cos, 16) || !aligned(sin, 16) || !aligned(len, 4)) return -6;
  kv_append_kernel<<<B, 128, 0, stream>>>((bf16x8*)qkv, (bf16x8*)kv, len, (const float4*)cos, (const float4*)sin, H, Hkv, D / 8,
                                          capacity);
  PB_CHECK_LAUNCH();
  return 0;
}

// Split-KV decode attention: out [B, H·D] bf16 for the rotated Q heads of qkv [B, (H + 2Hkv)·D] over kv [B, capacity, 2·Hkv·D].
// Row b sees keys max(lo[b], len[b] - window) <= k < len[b]; lo may be null (0), window 0 = none. part: fp32 [B, H, splits, D + 2]
// workspace of the second (combine) kernel; unused, and may be null, when splits == 1 (then one launch writes out directly).
PB_EXPORT int pb_decode_attn(const void* qkv, const void* kv, const int* len, const int* lo, int window, void* out, float* part, int B,
                             int H, int Hkv, int D, int capacity, int splits, float scale, cudaStream_t stream) {
  if (qkv == nullptr || kv == nullptr || len == nullptr || out == nullptr || (splits > 1 && part == nullptr)) return -1;
  if (D != 64 && D != 128) return -2;
  if (B < 1 || H < 1 || Hkv < 1 || capacity < 1 || H % Hkv != 0) return -3;
  if (window < 0) return -4;
  if (splits < 1) return -5;
  if (!aligned(qkv, 16) || !aligned(kv, 16) || !aligned(out, 16) || !aligned(len, 4) || !aligned(lo, 4) || !aligned(part, 4)) return -6;
  const int tiles = (capacity + kSplitKeys - 1) / kSplitKeys;
  DecodeParams p{(const __nv_bfloat16*)qkv, (const __nv_bfloat16*)kv, len, lo, (__nv_bfloat16*)out, part, H, Hkv, H / Hkv, 1,
                 capacity, window, splits, (tiles + splits - 1) / splits * kSplitKeys, scale * 1.4426950408889634f, 1};
  return D == 128 ? launch_attn<128, false, false>(p, B, stream) : launch_attn<64, false, false>(p, B, stream);
}

// The split policy of pb_decode_attn: a function of the cache geometry only, never of the lengths, so a decode step captured in a
// CUDA graph stays valid at every position. About two waves of CTAs over 132 SMs, at least 256 keys (four tiles) per split.
PB_EXPORT int pb_decode_attn_splits(int B, int Hkv, int capacity) {
  if (B < 1 || Hkv < 1 || capacity < 1) return -3;
  const int ctas = B * Hkv;
  int s = (2 * 132 + ctas - 1) / ctas;
  s = min(s, max(1, capacity / (4 * kSplitKeys)));
  return max(s, 1);
}

// ------------------------------------------------------------------------------------------------------- verify step (T tokens)
// Speculative decoding checks T = k + 1 tokens per row in one target forward. Same return codes as above, plus -3 for T < 1.

// At the start of a verify step, per row: the rule of pb_decode_advance applied to tokens[b, 0 .. T-1] in order, with the document
// start of each query written to lo_q [B, T] (int32); afterwards len += T, lo = lo_q[b, T-1], last_tok = tokens[b, T-1].
PB_EXPORT int pb_verify_advance(const int64_t* tokens, int T, int64_t eos, int* len, int* lo, int* lo_q, int64_t* last_tok, int B,
                                cudaStream_t stream) {
  if (tokens == nullptr || len == nullptr || lo == nullptr || lo_q == nullptr || last_tok == nullptr) return -1;
  if (B < 1 || T < 1) return -3;
  if (!aligned(tokens, 8) || !aligned(last_tok, 8) || !aligned(len, 4) || !aligned(lo, 4) || !aligned(lo_q, 4)) return -6;
  verify_advance_kernel<<<(B + 127) / 128, 128, 0, stream>>>(tokens, T, eos, len, lo, lo_q, last_tok, B);
  PB_CHECK_LAUNCH();
  return 0;
}

// qkv: the T new tokens' un-rotated fused rows [B, T, (H + 2Hkv)·D]; token t of row b is at position len[b] - T + t. As pb_kv_append
// per token: Q heads rotated in place, rotated K and V written to that cache row, positions outside [0, capacity) left alone.
PB_EXPORT int pb_kv_append_tokens(void* qkv, void* kv, const int* len, const float* cos, const float* sin, int B, int T, int H, int Hkv,
                                  int D, int capacity, cudaStream_t stream) {
  if (qkv == nullptr || kv == nullptr || len == nullptr || cos == nullptr || sin == nullptr) return -1;
  if (D != 64 && D != 128) return -2;
  if (B < 1 || T < 1 || H < 1 || Hkv < 1 || capacity < 1 || H % Hkv != 0) return -3;
  if (!aligned(qkv, 16) || !aligned(kv, 16) || !aligned(cos, 16) || !aligned(sin, 16) || !aligned(len, 4)) return -6;
  kv_append_tokens_kernel<<<dim3(T, B), 128, 0, stream>>>((bf16x8*)qkv, (bf16x8*)kv, len, (const float4*)cos, (const float4*)sin, T, H,
                                                          Hkv, D / 8, capacity);
  PB_CHECK_LAUNCH();
  return 0;
}

// Split-KV attention of T queries per row: out [B, T, H·D] bf16 for the rotated Q heads of qkv [B, T, (H + 2Hkv)·D] over kv. Query t
// of row b (position pos = len[b] - T + t) sees keys max(lo[b, t], pos + 1 - window) <= k <= pos, lo [B, T] nullable. part: fp32
// [B, T, H, splits, D + 2] when splits > 1. With T = 1 it computes exactly what pb_decode_attn computes, bit for bit.
PB_EXPORT int pb_verify_attn(const void* qkv, const void* kv, const int* len, const int* lo, int window, void* out, float* part, int B,
                             int T, int H, int Hkv, int D, int capacity, int splits, float scale, cudaStream_t stream) {
  if (qkv == nullptr || kv == nullptr || len == nullptr || out == nullptr || (splits > 1 && part == nullptr)) return -1;
  if (D != 64 && D != 128) return -2;
  if (B < 1 || T < 1 || H < 1 || Hkv < 1 || capacity < 1 || H % Hkv != 0) return -3;
  if (window < 0) return -4;
  if (splits < 1) return -5;
  if (!aligned(qkv, 16) || !aligned(kv, 16) || !aligned(out, 16) || !aligned(len, 4) || !aligned(lo, 4) || !aligned(part, 4)) return -6;
  const int tiles = (capacity + kSplitKeys - 1) / kSplitKeys;
  DecodeParams p{(const __nv_bfloat16*)qkv, (const __nv_bfloat16*)kv, len, lo, (__nv_bfloat16*)out, part, H, Hkv, H / Hkv, 1,
                 capacity, window, splits, (tiles + splits - 1) / splits * kSplitKeys, scale * 1.4426950408889634f, T};
  return D == 128 ? launch_attn<128, true, false>(p, B, stream) : launch_attn<64, true, false>(p, B, stream);
}

// ------------------------------------------------------------------------------------------------------------ e4m3 cache (fp8)
// The layout is the bf16 cache's in bytes, kv uint8 [B, capacity, 2·Hkv·D], plus kv_scale uint8 [B, capacity, 2·Hkv·D/32] (see the
// top of this file). Same return codes as above; a null kv_scale is -1, and kv_scale must be 4-byte and kv 8-byte aligned (-6).

// pb_kv_append_tokens into an e4m3 cache (T = 1: the decode step's append): Q heads rotated in place, then the rotated K (rounded
// to bf16) and V of each token quantised into its cache row.
PB_EXPORT int pb_kv_append_fp8(void* qkv, void* kv, void* kv_scale, const int* len, const float* cos, const float* sin, int B, int T, int H,
                               int Hkv, int D, int capacity, cudaStream_t stream) {
  if (qkv == nullptr || kv == nullptr || kv_scale == nullptr || len == nullptr || cos == nullptr || sin == nullptr) return -1;
  if (D != 64 && D != 128) return -2;
  if (B < 1 || T < 1 || H < 1 || Hkv < 1 || capacity < 1 || H % Hkv != 0) return -3;
  if (!aligned(qkv, 16) || !aligned(kv, 8) || !aligned(kv_scale, 4) || !aligned(cos, 16) || !aligned(sin, 16) || !aligned(len, 4)) return -6;
  kv_append_fp8_kernel<<<dim3(T, B), 128, 0, stream>>>((bf16x8*)qkv, (uint2*)kv, (uint8_t*)kv_scale, len, (const float4*)cos,
                                                       (const float4*)sin, T, H, Hkv, D / 8, capacity);
  PB_CHECK_LAUNCH();
  return 0;
}

// Prefill: quantise S bf16 rows per sequence, row (b, s) at src + (b·S + s)·src_row_stride elements and cols wide (the K|V columns
// of the fused QKV activation: src = qkv + H·D, stride (H + 2Hkv)·D), into rows 0 .. S-1 of the e4m3 cache. -3 for S > capacity
// or cols not a multiple of 32 or wider than the stride; src and its stride must keep 16-byte rows (-6).
PB_EXPORT int pb_kv_quantize(const void* src, int64_t src_row_stride, void* kv, void* kv_scale, int B, int S, int cols, int capacity,
                             cudaStream_t stream) {
  if (src == nullptr || kv == nullptr || kv_scale == nullptr) return -1;
  if (B < 1 || S < 1 || capacity < S || cols < 32 || cols % 32 != 0 || src_row_stride < cols) return -3;
  if (!aligned(src, 16) || src_row_stride % 8 != 0 || !aligned(kv, 8) || !aligned(kv_scale, 4)) return -6;
  const int64_t total = (int64_t)B * S * (cols / 8);
  const int grid = (int)std::min<int64_t>((total + 255) / 256, 132 * 16);
  kv_quantize_kernel<<<grid, 256, 0, stream>>>((const __nv_bfloat16*)src, src_row_stride, (uint2*)kv, (uint8_t*)kv_scale, S, cols / 8,
                                               capacity, total);
  PB_CHECK_LAUNCH();
  return 0;
}

// pb_decode_attn over an e4m3 cache. At the same split count its result is the bf16 kernel's math on the dequantised cache.
PB_EXPORT int pb_decode_attn_fp8(const void* qkv, const void* kv, const void* kv_scale, const int* len, const int* lo, int window, void* out,
                                 float* part, int B, int H, int Hkv, int D, int capacity, int splits, float scale, cudaStream_t stream) {
  if (qkv == nullptr || kv == nullptr || kv_scale == nullptr || len == nullptr || out == nullptr || (splits > 1 && part == nullptr)) return -1;
  if (D != 64 && D != 128) return -2;
  if (B < 1 || H < 1 || Hkv < 1 || capacity < 1 || H % Hkv != 0) return -3;
  if (window < 0) return -4;
  if (splits < 1) return -5;
  if (!aligned(qkv, 16) || !aligned(kv, 8) || !aligned(kv_scale, 4) || !aligned(out, 16) || !aligned(len, 4) || !aligned(lo, 4) ||
      !aligned(part, 4))
    return -6;
  const int tiles = (capacity + kSplitKeys - 1) / kSplitKeys;
  DecodeParams p{(const __nv_bfloat16*)qkv, (const __nv_bfloat16*)kv, len, lo, (__nv_bfloat16*)out, part, H, Hkv, H / Hkv, 1,
                 capacity, window, splits, (tiles + splits - 1) / splits * kSplitKeys, scale * 1.4426950408889634f, 1,
                 (const uint8_t*)kv_scale};
  return D == 128 ? launch_attn<128, false, true>(p, B, stream) : launch_attn<64, false, true>(p, B, stream);
}

// pb_verify_attn over an e4m3 cache; with T = 1 it computes exactly what pb_decode_attn_fp8 computes, bit for bit.
PB_EXPORT int pb_verify_attn_fp8(const void* qkv, const void* kv, const void* kv_scale, const int* len, const int* lo, int window, void* out,
                                 float* part, int B, int T, int H, int Hkv, int D, int capacity, int splits, float scale,
                                 cudaStream_t stream) {
  if (qkv == nullptr || kv == nullptr || kv_scale == nullptr || len == nullptr || out == nullptr || (splits > 1 && part == nullptr)) return -1;
  if (D != 64 && D != 128) return -2;
  if (B < 1 || T < 1 || H < 1 || Hkv < 1 || capacity < 1 || H % Hkv != 0) return -3;
  if (window < 0) return -4;
  if (splits < 1) return -5;
  if (!aligned(qkv, 16) || !aligned(kv, 8) || !aligned(kv_scale, 4) || !aligned(out, 16) || !aligned(len, 4) || !aligned(lo, 4) ||
      !aligned(part, 4))
    return -6;
  const int tiles = (capacity + kSplitKeys - 1) / kSplitKeys;
  DecodeParams p{(const __nv_bfloat16*)qkv, (const __nv_bfloat16*)kv, len, lo, (__nv_bfloat16*)out, part, H, Hkv, H / Hkv, 1,
                 capacity, window, splits, (tiles + splits - 1) / splits * kSplitKeys, scale * 1.4426950408889634f, T,
                 (const uint8_t*)kv_scale};
  return D == 128 ? launch_attn<128, true, true>(p, B, stream) : launch_attn<64, true, true>(p, B, stream);
}
