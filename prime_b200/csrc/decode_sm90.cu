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
#include <math.h>

#include "common.cuh"

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
// One token's fused row at position pos: Q heads are rotated in place, K heads are rotated into the cache row dst, V heads are
// copied; the rotation is rope_inplace_kernel's (interleaved pairs, fp32, one bf16 rounding).
__device__ __forceinline__ void append_row(bf16x8* __restrict__ row, bf16x8* __restrict__ dst, const float4* __restrict__ cosb,
                                           const float4* __restrict__ sinb, int pos, int H, int Hkv, int vec) {
  const int n = (H + 2 * Hkv) * vec;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int head = i / vec, vh = i - head * vec;
    bf16x8 x = row[i];
    if (head < H + Hkv) {
      float v[8], o[8];
      pb::unpack8(x, v);
      const float4 c = cosb[(int64_t)pos * vec + vh], s = sinb[(int64_t)pos * vec + vh];
      const float cc[4] = {c.x, c.y, c.z, c.w}, sn[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        o[2 * j] = v[2 * j] * cc[j] - v[2 * j + 1] * sn[j];
        o[2 * j + 1] = v[2 * j] * sn[j] + v[2 * j + 1] * cc[j];
      }
      x = pb::pack8(o);
    }
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
};

constexpr int kDecThreads = 128;
constexpr int kDecWarps = kDecThreads / 32;

// Grid (split, kv head × query chunk, row). A CTA owns GC <= 8 query vectors of one GQA group, so every K / V byte of its key range
// is read once per chunk of 8 query vectors. Decoding, the vectors are the chunk's heads of the group (G <= 8: once per step);
// verifying (kMulti), they are the (token t, head g) pairs j = t·G + g of the T·G queries of the group, each with its own key range,
// and the CTA's key loop covers the union of those ranges. A lane group of D/8 lanes holds one key, each lane 8 of its dimensions; a
// warp covers 32·8/D keys per load and every lane keeps kUnroll keys' K and V loads in flight. Scores are reduced over the lane group
// by shuffles; each lane group runs its own online softmax, and the groups are merged (shuffles, then shared memory) at the end.
template <int D, int GC, bool kMulti>
__device__ __forceinline__ void attn_body(const DecodeParams& p) {
  constexpr int LPK = D / 8;   // lanes per key
  constexpr int KPW = 32 / LPK;  // keys per warp and load
  constexpr int kUnroll = GC >= 8 ? 2 : 4;
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
    // the loop bound is uniform over the warp (the shuffles below need every lane); keys past k1 are loaded by no lane and score -inf
    for (int wb = k0 + warp * KPW * kUnroll; wb < k1; wb += KPI) {
      const int base = wb + grp;
      bf16x8 kr[kUnroll] = {}, vr[kUnroll] = {};
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int key = base + u * KPW;
        if (key < k1) {
          kr[u] = pb::ldg_stream(reinterpret_cast<const bf16x8*>(kbase + (int64_t)key * ldkv));
          vr[u] = pb::ldg_stream(reinterpret_cast<const bf16x8*>(vbase + (int64_t)key * ldkv));
        }
      }
      float s[kUnroll][GC];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        float kf[8];
        pb::unpack8(kr[u], kf);
#pragma unroll
        for (int g = 0; g < GC; ++g) {
          float d = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) d = fmaf(q[g][j], kf[j], d);
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
        pb::unpack8(vr[u], vf);
#pragma unroll
        for (int g = 0; g < GC; ++g) {
          l[g] += s[u][g];
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[g][j] = fmaf(s[u][g], vf[j], acc[g][j]);
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

template <int D>
int launch_decode(const DecodeParams& p0, int B, cudaStream_t stream) {
  DecodeParams p = p0;
  const int gc = p.G > 4 ? 8 : p.G > 2 ? 4 : p.G;  // smallest power of two >= G, at most 8 (G > 8: several chunks of 8)
  p.chunks = (p.G + gc - 1) / gc;
  const dim3 grid(p.splits, p.Hkv * p.chunks, B);
  if (gc == 8) decode_attn_kernel<D, 8><<<grid, kDecThreads, 0, stream>>>(p);
  else if (gc == 4) decode_attn_kernel<D, 4><<<grid, kDecThreads, 0, stream>>>(p);
  else if (gc == 2) decode_attn_kernel<D, 2><<<grid, kDecThreads, 0, stream>>>(p);
  else decode_attn_kernel<D, 1><<<grid, kDecThreads, 0, stream>>>(p);
  if (p.splits > 1) decode_combine_kernel<<<B * p.H, 128, 0, stream>>>(p.part, p.out, p.H, D, p.splits);
  PB_CHECK_LAUNCH();
  return 0;
}

// The verify step: T·G query vectors per KV group, in chunks of the smallest power of two >= T·G, at most 8.
template <int D>
int launch_verify(const DecodeParams& p0, int B, cudaStream_t stream) {
  DecodeParams p = p0;
  const int nq = p.T * p.G;
  const int gc = nq > 4 ? 8 : nq > 2 ? 4 : nq;
  p.chunks = (nq + gc - 1) / gc;
  const dim3 grid(p.splits, p.Hkv * p.chunks, B);
  if (gc == 8) verify_attn_kernel<D, 8><<<grid, kDecThreads, 0, stream>>>(p);
  else if (gc == 4) verify_attn_kernel<D, 4><<<grid, kDecThreads, 0, stream>>>(p);
  else if (gc == 2) verify_attn_kernel<D, 2><<<grid, kDecThreads, 0, stream>>>(p);
  else verify_attn_kernel<D, 1><<<grid, kDecThreads, 0, stream>>>(p);
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
  return D == 128 ? launch_decode<128>(p, B, stream) : launch_decode<64>(p, B, stream);
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
  return D == 128 ? launch_verify<128>(p, B, stream) : launch_verify<64>(p, B, stream);
}
