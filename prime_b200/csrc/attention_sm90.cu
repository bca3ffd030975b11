// Flash attention for sm_90a on the fused QKV activation, forward and backward, with bf16 mma.sync tensor-core tiles.
//
//   qkv  [B, S, (H + 2·Hkv)·D] bf16: Q heads, then K heads, then V heads of every token (GQA: Q head h reads KV head h / (H/Hkv))
//   out  [B, S, H·D] bf16
//   lse2 [B, H, S] fp32 = log2-domain log-sum-exp of (scale·log2e·s), consumed by the backward kernels
//
// Forward (flash_fwd_kernel): one CTA of 4 warps per (64-query block, b, h); every warp owns 16 query rows, keeps Q in registers
// and runs the online softmax over 64-key tiles that are double-buffered in shared memory with cp.async.
// Backward (deterministic, no atomics):
//   delta[b,h,s] = Σ_d dO·O · scale                                                      (bwd_delta_kernel, memory bound)
//   dK, dV: one CTA per (64-key block, b, kv head); loops over the heads of the group and 32-query tiles, computing the
//           TRANSPOSED scores Sᵀ = K Qᵀ and dPᵀ = V dOᵀ so that each warp owns 16 key rows:  dV += Pᵀ dO,  dK += dSᵀ Q
//   dQ:     one CTA per (64-query block, b, h); loops over 64-key tiles: S = Q Kᵀ, dP = dO Vᵀ,  dQ += dS K
// With dS = P ∘ (dP·scale − delta·scale) the results need no further scaling; P is recomputed from lse2.
// Optional RoPE backward (non-null rope_cos / rope_sin of pb_flash_attn_bwd): the inverse rotation is applied to dQ / dK in registers
// before the store.
// Optional lower-bounded causal masking (kDoc, selected by a non-null doc_start): query q of row b sees key k iff
// lo[q] <= k <= q, where lo = doc_start is any int32 [B, S] array that never decreases along a row and has lo[q] <= q, and
// end = doc_end is its matching upper bound (end[k] = one past the last query that sees key k). pb_doc_bounds builds them for
// documents of packed rows, a sliding window of W keys (lo[q] = q - W + 1), or both. Key tiles below a query block's first
// visible key are skipped, not masked.
#include <type_traits>

#include "common.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int kThreads = 128;
constexpr int BQ = 64;    // forward / dQ query block
constexpr int BKV = 64;   // key block
constexpr int BQB = 32;   // query tile of the dK/dV kernel

// Shared-memory tile of `rows` x D bf16 with a 16-byte pad per row (conflict-free ldmatrix).
template <int D>
struct Tile {
  static constexpr int kLd = D + 8;  // elements per row
  __host__ __device__ static constexpr uint32_t bytes(int rows) { return (uint32_t)rows * kLd * 2; }
};

// rows x D bf16 from global (row stride ld elements) into a padded tile, 16 B per cp.async
template <int D>
__device__ __forceinline__ void load_tile(uint32_t dst, const __nv_bfloat16* src, int64_t ld, int rows) {
  constexpr int kChunks = D / 8;
  for (int i = threadIdx.x; i < rows * kChunks; i += kThreads) {
    const int r = i / kChunks, c = i - r * kChunks;
    cp_async16(dst + (uint32_t)(r * Tile<D>::kLd + c * 8) * 2, src + r * ld + c * 8);
  }
}

// A operand (16 rows x 16 k) at (row0, k0) of a padded row-major tile
template <int D>
__device__ __forceinline__ void ld_a(uint32_t base, int row0, int k0, uint32_t (&a)[4]) {
  const int l = threadIdx.x & 31;
  ldsm_x4(base + (uint32_t)((row0 + (l & 15)) * Tile<D>::kLd + k0 + (l >> 4) * 8) * 2, a);
}

// Tile products, one k16 step each: acc[n] += A · B[k0 .. k0 + 16, 8n .. 8n + 8] for every n8 block of acc, where A is a 16 x 16
// fragment (ld_a). Callers step k0 upwards, so every accumulator adds its products in increasing k.
// B stored [n][k] (k contiguous): the K tile of Q·Kᵀ, the Q tile of K·Qᵀ.
template <int D, int N8>
__device__ __forceinline__ void mma_b_nk(float (&acc)[N8][4], const uint32_t (&a)[4], uint32_t b, int k0) {
  const int l = threadIdx.x & 31;
#pragma unroll
  for (int n = 0; n < N8; n += 2) {
    uint32_t bf[4];
    ldsm_x4(b + (uint32_t)((n * 8 + (l & 7) + (l >> 4) * 8) * Tile<D>::kLd + k0 + ((l >> 3) & 1) * 8) * 2, bf);
    mma16816(acc[n], a, bf[0], bf[1]);
    mma16816(acc[n + 1], a, bf[2], bf[3]);
  }
}
// B stored [k][n] (n contiguous): the V tile of P·V, the K tile of dS·K.
template <int D, int N8>
__device__ __forceinline__ void mma_b_kn(float (&acc)[N8][4], const uint32_t (&a)[4], uint32_t b, int k0) {
  const int l = threadIdx.x & 31;
#pragma unroll
  for (int n = 0; n < N8; n += 2) {
    uint32_t bf[4];
    ldsm_x4_t(b + (uint32_t)((k0 + (l & 7) + ((l >> 3) & 1) * 8) * Tile<D>::kLd + n * 8 + (l >> 4) * 8) * 2, bf);
    mma16816(acc[n], a, bf[0], bf[1]);
    mma16816(acc[n + 1], a, bf[2], bf[3]);
  }
}

struct AttnParams {
  const __nv_bfloat16* qkv;
  __nv_bfloat16* out;
  const __nv_bfloat16* dout;
  __nv_bfloat16* dqkv;
  const float* lse2;   // [B, H, S]
  const float* delta;  // [B, H, S], rowsum(dO∘O) · scale
  float* lse2_out;
  int B, S, H, Hkv;
  float scale, scale_log2;
  int causal;
  const float* rope_cos;  // backward only: fp32 [S, D/2] tables of the forward rotation, nullptr = no RoPE
  const float* rope_sin;
  const int* doc_start;  // kDoc kernels only: int32 [B, S] lo[s], the first key query s sees (non-decreasing, <= s)
  const int* doc_end;    //                     int32 [B, S] end[s], one past the last query that sees key s
};

// One batch row of the fused [B, S, (H + 2·Hkv)·D] activation (qkv, or its gradient dqkv): the Q head h, K head hk and V head hk
// of token s.
template <int D, typename T>
struct FusedRow {
  T* row;  // token 0
  int W;   // elements per token
  int H, Hkv;
  __device__ FusedRow(T* x, const AttnParams& p, int b)
      : row(x + (int64_t)b * p.S * ((p.H + 2 * p.Hkv) * D)), W((p.H + 2 * p.Hkv) * D), H(p.H), Hkv(p.Hkv) {}
  __device__ T* q(int s, int h) const { return row + (int64_t)s * W + h * D; }
  __device__ T* k(int s, int hk) const { return q(s, H + hk); }
  __device__ T* v(int s, int hk) const { return q(s, H + Hkv + hk); }
};

// Which keys the queries of one batch row see: all of them when not causal, k <= q when causal, and lo[q] <= k <= q under kDoc
// (which implies causal). lo never decreases along a row and end is its matching upper bound, so the keys a block of queries sees
// and the queries that see a block of keys are contiguous tile ranges: the kernels skip the tiles outside them, and only edge
// tiles pay for the per-element predicate. Built once per block; kDoc = false never reads the bounds.
template <bool kDoc>
struct Visibility {
  const int* lo;  // kDoc: doc_start of the row
  bool causal;
  int first, end;  // the tiles the block visits: key tiles of a query block, query tiles of a key block
  int qb;          // query block: its index, whose key tile holds the diagonal
  int lo_last;     // query block, kDoc: lo of its last query; key tiles below it hold keys some query of the block does not see

  // 64-key tiles [first, end) that 64-query block qb sees something of
  __device__ static Visibility query_block(const AttnParams& p, int b, int qb) {
    Visibility v{kDoc ? p.doc_start + (int64_t)b * p.S : nullptr, p.causal != 0};
    v.qb = qb;
    v.first = kDoc ? v.lo[qb * BQ] / BKV : 0;
    v.end = p.causal ? qb + 1 : p.S / BKV;
    v.lo_last = kDoc ? v.lo[qb * BQ + BQ - 1] : 0;
    return v;
  }
  // 32-query tiles [first, end) that see something of 64-key block kb (end stops at the tile holding end[last key of the block])
  __device__ static Visibility key_block(const AttnParams& p, int b, int kb) {
    Visibility v{kDoc ? p.doc_start + (int64_t)b * p.S : nullptr, p.causal != 0};
    v.first = p.causal ? kb * BKV / BQB : 0;
    v.end = kDoc ? (p.doc_end[(int64_t)b * p.S + kb * BKV + BKV - 1] + BQB - 1) / BQB : p.S / BQB;
    return v;
  }
  __device__ int lo_of(int q) const { return kDoc ? lo[q] : 0; }
  // query block: key tile j is the diagonal tile or lies below lo_last
  __device__ bool masked(int j) const { return causal && (j == qb || (kDoc && j * BKV < lo_last)); }
  // query q sees key k; lo_q = lo_of(q), which the kernels keep in registers or shared memory
  __device__ bool sees(int q, int k, int lo_q) const { return kDoc ? lo_q <= k && k <= q : !causal || k <= q; }
};

// ------------------------------------------------------------------------------------------------------------------ forward
// The key loop starts at Visibility::first, whose tile the first cp.async prefetch loads.
template <int D, bool kDoc>
__global__ void __launch_bounds__(kThreads) flash_fwd_kernel(const AttnParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int qb = (int)blockIdx.x, bh = (int)blockIdx.y;
  const int b = bh / p.H, h = bh - b * p.H, hk = h / (p.H / p.Hkv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const FusedRow<D, const __nv_bfloat16> x(p.qkv, p, b);
  const uint32_t sq = smem_u32(smem);
  const uint32_t skv = sq + Tile<D>::bytes(BQ);  // [stage][K | V]
  constexpr uint32_t kKV = Tile<D>::bytes(BKV);

  const int q0 = qb * BQ;
  const auto vis = Visibility<kDoc>::query_block(p, b, qb);
  const int rlo[2] = {vis.lo_of(q0 + warp * 16 + g), vis.lo_of(q0 + warp * 16 + g + 8)};  // this thread's two rows
  load_tile<D>(sq, x.q(q0, h), x.W, BQ);
  load_tile<D>(skv, x.k(vis.first * BKV, hk), x.W, BKV);
  load_tile<D>(skv + kKV, x.v(vis.first * BKV, hk), x.W, BKV);
  cp_async_commit();

  uint32_t qf[D / 16][4];
  float o[D / 8][4] = {};
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

  for (int j = vis.first; j < vis.end; ++j) {
    const int st = (j - vis.first) & 1;
    if (j + 1 < vis.end) {  // prefetch the next key/value tile into the other stage
      const int k1 = (j + 1) * BKV;
      const uint32_t nxt = skv + (st ^ 1) * 2 * kKV;
      load_tile<D>(nxt, x.k(k1, hk), x.W, BKV);
      load_tile<D>(nxt + kKV, x.v(k1, hk), x.W, BKV);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    if (j == vis.first) {
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) ld_a<D>(sq, warp * 16, kk * 16, qf[kk]);
    }
    const uint32_t sk = skv + st * 2 * kKV, sv = sk + kKV;
    float s[BKV / 8][4] = {};
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) mma_b_nk<D>(s, qf[kk], sk, kk * 16);
    // online softmax (log2 domain); rows g and g + 8 of this warp's 16
    const bool masked = vis.masked(j);
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = e >> 1;
        float v = s[n][e] * p.scale_log2;
        if (masked) {
          const int qi = warp * 16 + g + r * 8, ki = n * 8 + 2 * t + (e & 1);
          // plain causal masks the diagonal tile only, where positions within the tile compare as token positions do. They do not
          // change with j; from token positions, the plain D = 128 forward compiles to 50 fewer registers and runs ~15 % slower.
          if (!(kDoc ? vis.sees(q0 + qi, j * BKV + ki, rlo[r]) : vis.sees(qi, ki, 0))) v = -INFINITY;
        }
        s[n][e] = v;
        mx[r] = fmaxf(mx[r], v);
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float corr[2], rs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if constexpr (kDoc) {
        // a row whose lower bound lies later in the block can meet tiles in which every key is masked; while its maximum is
        // still -inf, subtract 0 so that exp2 gives 0 instead of exp2(-inf - -inf) = NaN (m is reset to -inf below)
        const float mref = mx[r] == -INFINITY ? 0.f : mx[r];
        corr[r] = fast_exp2(m[r] - mref);
        m[r] = mref;
      } else {
        corr[r] = fast_exp2(m[r] - mx[r]);  // m = -inf on the first tile → 0
        m[r] = mx[r];
      }
    }
    uint32_t pf[BKV / 16][4];
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
      const float e0 = fast_exp2(s[n][0] - m[0]), e1 = fast_exp2(s[n][1] - m[0]);
      const float e2 = fast_exp2(s[n][2] - m[1]), e3 = fast_exp2(s[n][3] - m[1]);
      rs[0] += e0 + e1;
      rs[1] += e2 + e3;
      pf[n >> 1][(n & 1) * 2] = pack_bf16(e0, e1);
      pf[n >> 1][(n & 1) * 2 + 1] = pack_bf16(e2, e3);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l[r] = l[r] * corr[r] + rs[r];
    if constexpr (kDoc) {
#pragma unroll
      for (int r = 0; r < 2; ++r) m[r] = mx[r];
    }
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      o[i][0] *= corr[0];
      o[i][1] *= corr[0];
      o[i][2] *= corr[1];
      o[i][3] *= corr[1];
    }
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) mma_b_kn<D>(o, pf[kk], sv, kk * 16);
    __syncthreads();  // this stage is refilled by the prefetch of iteration j + 1
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
  const float inv[2] = {1.f / l[0], 1.f / l[1]};
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + warp * 16 + g + r * 8;
    __nv_bfloat16* dst = p.out + ((int64_t)b * p.S + q) * (p.H * D) + h * D + 2 * t;
#pragma unroll
    for (int n = 0; n < D / 8; ++n)
      *reinterpret_cast<uint32_t*>(dst + n * 8) = pack_bf16(o[n][2 * r] * inv[r], o[n][2 * r + 1] * inv[r]);
    if (t == 0) p.lse2_out[(int64_t)bh * p.S + q] = m[r] + log2f(l[r]);
  }
}

// ------------------------------------------------------------------------------------------------------------------ backward
__global__ void __launch_bounds__(256) bwd_delta_kernel(const pb::bf16x8* __restrict__ dout, const pb::bf16x8* __restrict__ out,
                                                        float* __restrict__ delta, int64_t tokens, int S, int H, int vec_per_head,
                                                        float scale) {
  // one warp per TOKEN: it walks the token's H·D row in fully coalesced 512-byte steps (32 lanes x 16 B) and reduces inside groups
  // of `vec_per_head` lanes (D = 128 → 16 lanes, two heads per step; D = 64 → 8 lanes, four heads per step).
  // Writes delta·scale (the only form the two kernels below use).
  const int64_t tok = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (tok >= tokens) return;
  const int vec_per_tok = H * vec_per_head;
  const int64_t base = tok * vec_per_tok;
  const int64_t bidx = tok / S;
  const int s = (int)(tok - bidx * S);
  for (int i0 = 0; i0 < vec_per_tok; i0 += 32) {
    const int i = i0 + lane;
    float acc = 0.f;
    if (i < vec_per_tok) {
      float a[8], c[8];
      pb::unpack8(pb::ldg_stream(dout + base + i), a);
      pb::unpack8(pb::ldg_stream(out + base + i), c);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc += a[j] * c[j];
    }
    for (int o = vec_per_head >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((lane & (vec_per_head - 1)) == 0 && i < vec_per_tok) {
      const int h = i / vec_per_head;
      delta[(bidx * H + h) * S + s] = acc * scale;
    }
  }
}

// store a 16-row x D fp32 accumulator (mma C layout) as bf16 into the 16 rows from dst on (row stride ld; token s0 first),
// optionally un-rotating the interleaved RoPE pairs (position = token)
template <int D>
__device__ __forceinline__ void store_rows(__nv_bfloat16* dst, int64_t ld, int s0, float (&acc)[D / 8][4], const AttnParams& p, bool rope) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = g + r * 8, pos = s0 + row;
#pragma unroll
    for (int n = 0; n < D / 8; ++n) {
      float a = acc[n][2 * r], c = acc[n][2 * r + 1];
      if (rope) {  // rotation is orthogonal: its backward is the inverse rotation
        const int64_t ti = (int64_t)pos * (D / 2) + n * 4 + t;
        const float cs = __ldg(p.rope_cos + ti), sn = __ldg(p.rope_sin + ti);
        const float x = a, y = c;
        a = x * cs + y * sn;
        c = -x * sn + y * cs;
      }
      *reinterpret_cast<uint32_t*>(dst + (int64_t)row * ld + n * 8 + 2 * t) = pack_bf16(a, c);
    }
  }
}

// The query-tile loop covers Visibility::key_block; the tile's lo values are staged in shared memory after lse2 and delta.
template <int D, bool kDoc>
__global__ void __launch_bounds__(kThreads) bwd_dkdv_kernel(const AttnParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int kb = (int)blockIdx.x, bhk = (int)blockIdx.y;
  const int b = bhk / p.Hkv, hk = bhk - b * p.Hkv, grp = p.H / p.Hkv;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const FusedRow<D, const __nv_bfloat16> x(p.qkv, p, b);
  const __nv_bfloat16* dbase = p.dout + (int64_t)b * p.S * (p.H * D);
  const uint32_t sk = smem_u32(smem), sv = sk + Tile<D>::bytes(BKV);
  const uint32_t sq = sv + Tile<D>::bytes(BKV), sdo = sq + Tile<D>::bytes(BQB);
  float* s_ld = reinterpret_cast<float*>(smem + 2 * Tile<D>::bytes(BKV) + 2 * Tile<D>::bytes(BQB));  // [lse2 BQB | delta BQB]
  int* s_lo = reinterpret_cast<int*>(s_ld + 2 * BQB);  // kDoc: [lo BQB]
  const int k0 = kb * BKV;
  load_tile<D>(sk, x.k(k0, hk), x.W, BKV);
  load_tile<D>(sv, x.v(k0, hk), x.W, BKV);
  cp_async_commit();

  float dk[D / 8][4] = {}, dv[D / 8][4] = {};
  const auto vis = Visibility<kDoc>::key_block(p, b, kb);
  for (int hh = 0; hh < grp; ++hh) {
    const int h = hk * grp + hh;
    for (int qt = vis.first; qt < vis.end; ++qt) {
      const int q0 = qt * BQB;
      __syncthreads();  // the previous tile has been consumed
      load_tile<D>(sq, x.q(q0, h), x.W, BQB);
      load_tile<D>(sdo, dbase + (int64_t)q0 * (p.H * D) + h * D, p.H * D, BQB);
      cp_async_commit();
      if (threadIdx.x < BQB) s_ld[threadIdx.x] = p.lse2[((int64_t)b * p.H + h) * p.S + q0 + threadIdx.x];
      else if (threadIdx.x < 2 * BQB) s_ld[threadIdx.x] = p.delta[((int64_t)b * p.H + h) * p.S + q0 + threadIdx.x - BQB];
      if constexpr (kDoc) {
        if (threadIdx.x >= 2 * BQB && threadIdx.x < 3 * BQB) s_lo[threadIdx.x - 2 * BQB] = vis.lo_of(q0 + threadIdx.x - 2 * BQB);
      }
      cp_async_wait<0>();
      __syncthreads();
      // Sᵀ = K Qᵀ and dPᵀ = V dOᵀ: 16 keys (this warp) x BQB queries
      float st[BQB / 8][4] = {}, dpt[BQB / 8][4] = {};
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        uint32_t ka[4], va[4];
        ld_a<D>(sk, warp * 16, kk * 16, ka);
        ld_a<D>(sv, warp * 16, kk * 16, va);
        mma_b_nk<D>(st, ka, sq, kk * 16);
        mma_b_nk<D>(dpt, va, sdo, kk * 16);
      }
      // Pᵀ = exp2(s·scale·log2e − lse2[q]) (0 where q does not see the key), dSᵀ = Pᵀ ∘ (dPᵀ·scale − delta·scale)
      uint32_t pa[BQB / 16][4], da[BQB / 16][4];
#pragma unroll
      for (int n = 0; n < BQB / 8; ++n) {
        float pv[4], dsv[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qi = n * 8 + 2 * t + (e & 1), ki = k0 + warp * 16 + g + (e >> 1) * 8;
          float pe = fast_exp2(st[n][e] * p.scale_log2 - s_ld[qi]);
          if (!vis.sees(q0 + qi, ki, kDoc ? s_lo[qi] : 0)) pe = 0.f;
          pv[e] = pe;
          dsv[e] = pe * (dpt[n][e] * p.scale - s_ld[BQB + qi]);
        }
        pa[n >> 1][(n & 1) * 2] = pack_bf16(pv[0], pv[1]);
        pa[n >> 1][(n & 1) * 2 + 1] = pack_bf16(pv[2], pv[3]);
        da[n >> 1][(n & 1) * 2] = pack_bf16(dsv[0], dsv[1]);
        da[n >> 1][(n & 1) * 2 + 1] = pack_bf16(dsv[2], dsv[3]);
      }
      // dV += Pᵀ dO, dK += dSᵀ Q  (k = queries)
#pragma unroll
      for (int kk = 0; kk < BQB / 16; ++kk) {
        mma_b_kn<D>(dv, pa[kk], sdo, kk * 16);
        mma_b_kn<D>(dk, da[kk], sq, kk * 16);
      }
    }
  }
  const FusedRow<D, __nv_bfloat16> dx(p.dqkv, p, b);
  const int s0 = k0 + warp * 16;
  store_rows<D>(dx.k(s0, hk), dx.W, s0, dk, p, p.rope_cos != nullptr);
  store_rows<D>(dx.v(s0, hk), dx.W, s0, dv, p, false);
}

// The key loop covers Visibility::query_block, masked as in the forward.
template <int D, bool kDoc>
__global__ void __launch_bounds__(kThreads) bwd_dq_kernel(const AttnParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int qb = (int)blockIdx.x, bh = (int)blockIdx.y;
  const int b = bh / p.H, h = bh - b * p.H, hk = h / (p.H / p.Hkv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const FusedRow<D, const __nv_bfloat16> x(p.qkv, p, b);
  const uint32_t sq = smem_u32(smem), sdo = sq + Tile<D>::bytes(BQ);
  const uint32_t sk = sdo + Tile<D>::bytes(BQ), sv = sk + Tile<D>::bytes(BKV);
  const int q0 = qb * BQ;
  load_tile<D>(sq, x.q(q0, h), x.W, BQ);
  load_tile<D>(sdo, p.dout + ((int64_t)b * p.S + q0) * (p.H * D) + h * D, p.H * D, BQ);
  cp_async_commit();
  float lse[2], del[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int64_t i = (int64_t)bh * p.S + q0 + warp * 16 + g + r * 8;
    lse[r] = p.lse2[i];
    del[r] = p.delta[i];
  }
  float dq[D / 8][4] = {};
  const auto vis = Visibility<kDoc>::query_block(p, b, qb);
  const int rlo[2] = {vis.lo_of(q0 + warp * 16 + g), vis.lo_of(q0 + warp * 16 + g + 8)};
  for (int j = vis.first; j < vis.end; ++j) {
    const int k0 = j * BKV;
    const bool masked = vis.masked(j);
    __syncthreads();
    load_tile<D>(sk, x.k(k0, hk), x.W, BKV);
    load_tile<D>(sv, x.v(k0, hk), x.W, BKV);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    float s[BKV / 8][4] = {}, dp[BKV / 8][4] = {};
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      uint32_t qa[4], oa[4];
      ld_a<D>(sq, warp * 16, kk * 16, qa);
      ld_a<D>(sdo, warp * 16, kk * 16, oa);
      mma_b_nk<D>(s, qa, sk, kk * 16);
      mma_b_nk<D>(dp, oa, sv, kk * 16);
    }
    uint32_t da[BKV / 16][4];
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
      float dsv[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = e >> 1, qi = q0 + warp * 16 + g + r * 8, ki = k0 + n * 8 + 2 * t + (e & 1);
        float pe = fast_exp2(s[n][e] * p.scale_log2 - lse[r]);
        if (masked && !vis.sees(qi, ki, rlo[r])) pe = 0.f;
        dsv[e] = pe * (dp[n][e] * p.scale - del[r]);
      }
      da[n >> 1][(n & 1) * 2] = pack_bf16(dsv[0], dsv[1]);
      da[n >> 1][(n & 1) * 2 + 1] = pack_bf16(dsv[2], dsv[3]);
    }
    // dQ += dS K  (k = keys)
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) mma_b_kn<D>(dq, da[kk], sk, kk * 16);
  }
  const FusedRow<D, __nv_bfloat16> dx(p.dqkv, p, b);
  store_rows<D>(dx.q(q0 + warp * 16, h), dx.W, q0 + warp * 16, dq, p, p.rope_cos != nullptr);
}

template <typename K>
int set_smem(K kernel, uint32_t bytes) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  return e == cudaSuccess ? 0 : (int)e;
}

template <int D, bool kDoc>
int launch_fwd(const AttnParams& p, cudaStream_t stream) {
  constexpr uint32_t kSmem = Tile<D>::bytes(BQ) + 4 * Tile<D>::bytes(BKV);
  static int rc = set_smem(flash_fwd_kernel<D, kDoc>, kSmem);
  if (rc) return rc;
  flash_fwd_kernel<D, kDoc><<<dim3(p.S / BQ, p.B * p.H), kThreads, kSmem, stream>>>(p);
  PB_CHECK_LAUNCH();
  return 0;
}

template <int D, bool kDoc>
int launch_bwd(const AttnParams& p, cudaStream_t stream) {
  const int64_t tokens = (int64_t)p.B * p.S;
  const int64_t blocks = (tokens * 32 + 255) / 256;
  bwd_delta_kernel<<<(unsigned)blocks, 256, 0, stream>>>((const pb::bf16x8*)p.dout, (const pb::bf16x8*)p.out, const_cast<float*>(p.delta),
                                                         tokens, p.S, p.H, D / 8, p.scale);
  PB_CHECK_LAUNCH();
  constexpr uint32_t kDkv = 2 * Tile<D>::bytes(BKV) + 2 * Tile<D>::bytes(BQB) + (kDoc ? 3 : 2) * BQB * 4;
  constexpr uint32_t kDq = 2 * Tile<D>::bytes(BQ) + 2 * Tile<D>::bytes(BKV);
  static int rc = set_smem(bwd_dkdv_kernel<D, kDoc>, kDkv) | set_smem(bwd_dq_kernel<D, kDoc>, kDq);
  if (rc) return rc;
  bwd_dkdv_kernel<D, kDoc><<<dim3(p.S / BKV, p.B * p.Hkv), kThreads, kDkv, stream>>>(p);
  bwd_dq_kernel<D, kDoc><<<dim3(p.S / BQ, p.B * p.H), kThreads, kDq, stream>>>(p);
  PB_CHECK_LAUNCH();
  return 0;
}

// launch(D, kDoc), both as std::integral_constant, for D ∈ {64, 128}; -2 for any other D
template <typename Launch>
int dispatch(int D, bool doc, Launch launch) {
  using D64 = std::integral_constant<int, 64>;
  using D128 = std::integral_constant<int, 128>;
  if (D == 128) return doc ? launch(D128(), std::true_type()) : launch(D128(), std::false_type());
  if (D == 64) return doc ? launch(D64(), std::true_type()) : launch(D64(), std::false_type());
  return -2;
}

// the fields both entry points set; the others stay null
AttnParams shared_params(const void* qkv, const int* doc_start, int B, int S, int H, int Hkv, float scale, int causal) {
  AttnParams p{};
  p.qkv = (const __nv_bfloat16*)qkv;
  p.doc_start = doc_start;
  p.B = B, p.S = S, p.H = H, p.Hkv = Hkv;
  p.scale = scale, p.scale_log2 = scale * 1.4426950408889634f;
  p.causal = causal;
  return p;
}

// Document bounds of packed rows: one CTA per row. Every thread owns a contiguous run of positions; a block-wide exclusive
// max-scan of the last document start per run (and min-scan, from the right, of the first EOS end) gives each run its carry-in.
// The window (1 <= window <= S; S = none) clamps both bounds as they are written.
constexpr int kBoundsThreads = 256;
__global__ void __launch_bounds__(kBoundsThreads) doc_bounds_kernel(const int64_t* __restrict__ tokens, int S, int64_t eos, int window,
                                                                    int* __restrict__ doc_start, int* __restrict__ doc_end) {
  constexpr int kWarps = kBoundsThreads / 32;
  __shared__ int s_lo[kWarps], s_hi[kWarps];
  const int64_t row = (int64_t)blockIdx.x * S;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per = (S + kBoundsThreads - 1) / kBoundsThreads;
  const int s0 = min(S, (int)threadIdx.x * per), s1 = min(S, s0 + per);
  int lo = 0, hi = S;  // last document start in [s0, s1), first end (EOS position + 1) in [s0, s1)
  for (int s = s0; s < s1; ++s)
    if (s > 0 && tokens[row + s - 1] == eos) lo = s;
  for (int s = s1 - 1; s >= s0; --s)
    if (tokens[row + s] == eos) hi = s + 1;
  int in_lo = lo, in_hi = hi;  // inclusive warp scans: max from the left, min from the right
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, in_lo, o), c = __shfl_down_sync(0xffffffffu, in_hi, o);
    if (lane >= o) in_lo = max(in_lo, a);
    if (lane + o < 32) in_hi = min(in_hi, c);
  }
  if (lane == 31) s_lo[warp] = in_lo;
  if (lane == 0) s_hi[warp] = in_hi;
  __syncthreads();
  int cur_lo = __shfl_up_sync(0xffffffffu, in_lo, 1), cur_hi = __shfl_down_sync(0xffffffffu, in_hi, 1);
  if (lane == 0) cur_lo = 0;
  if (lane == 31) cur_hi = S;
  for (int w = 0; w < warp; ++w) cur_lo = max(cur_lo, s_lo[w]);
  for (int w = warp + 1; w < kWarps; ++w) cur_hi = min(cur_hi, s_hi[w]);
  for (int s = s0; s < s1; ++s) {
    if (s > 0 && tokens[row + s - 1] == eos) cur_lo = s;
    doc_start[row + s] = max(cur_lo, s - window + 1);
  }
  for (int s = s1 - 1; s >= s0; --s) {
    if (tokens[row + s] == eos) cur_hi = s + 1;
    doc_end[row + s] = min(cur_hi, s + window);
  }
}

}  // namespace

// qkv [B, S, (H+2Hkv)·D] → out [B, S, H·D], lse2 [B, H, S].  S % 128 == 0, D ∈ {64, 128}.
// doc_start: null, or an int32 [B, S] lower bound lo (non-decreasing along a row, lo[q] <= q; pb_doc_bounds builds it for documents
// and / or a sliding window) for masked causal attention (causal != 0): query q attends key k iff doc_start[b, q] <= k <= q.
PB_EXPORT int pb_flash_attn_fwd(const void* qkv, void* out, float* lse2, const int* doc_start, int B, int S, int H, int Hkv, int D,
                                float scale, int causal, cudaStream_t stream) {
  if (S % 128 != 0 || H % Hkv != 0 || (doc_start != nullptr && !causal)) return -1;
  AttnParams p = shared_params(qkv, doc_start, B, S, H, Hkv, scale, causal);
  p.out = (__nv_bfloat16*)out;
  p.lse2_out = lse2;
  return dispatch(D, doc_start != nullptr,
                  [&](auto d, auto doc) { return launch_fwd<decltype(d)::value, decltype(doc)::value>(p, stream); });
}

// delta: [B, H, S] fp32 scratch.  dqkv: [B, S, (H+2Hkv)·D] bf16, fully overwritten.
// doc_start / doc_end: both null, or both the forward's lower bound and its matching upper bound (causal != 0).
// rope_cos / rope_sin: null, or the fp32 [S, D/2] tables of a forward rotation, whose inverse is fused into the dQ / dK stores.
PB_EXPORT int pb_flash_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta, void* dqkv,
                                const int* doc_start, const int* doc_end, int B, int S, int H, int Hkv, int D, float scale, int causal,
                                const float* rope_cos, const float* rope_sin, cudaStream_t stream) {
  if (S % 128 != 0 || H % Hkv != 0 || (doc_start == nullptr) != (doc_end == nullptr) || (doc_start != nullptr && !causal)) return -1;
  AttnParams p = shared_params(qkv, doc_start, B, S, H, Hkv, scale, causal);
  p.out = (__nv_bfloat16*)out;
  p.dout = (const __nv_bfloat16*)dout;
  p.dqkv = (__nv_bfloat16*)dqkv;
  p.lse2 = lse2;
  p.delta = delta;
  p.rope_cos = rope_cos, p.rope_sin = rope_sin;
  p.doc_end = doc_end;
  return dispatch(D, doc_start != nullptr,
                  [&](auto d, auto doc) { return launch_bwd<decltype(d)::value, decltype(doc)::value>(p, stream); });
}

// tokens int64 [B, S] → doc_start, doc_end int32 [B, S], the lo / end bounds of pb_flash_attn_fwd / _bwd. Position s starts a
// document when s == 0 or tokens[b, s-1] == eos; eos < 0 means no documents (token ids are never negative). window: 0 = none,
// else query s sees only the `window` most recent keys, itself included. Query s attends key k iff lo[s] <= k <= s with
// lo[s] = max(first position of the document holding s, s - window + 1), and end[s] = min(one past the document's last position
// (after its EOS, or S), s + window) is one past the last query that sees key s.
PB_EXPORT int pb_doc_bounds(const int64_t* tokens, int B, int S, int64_t eos, int window, int* doc_start, int* doc_end,
                            cudaStream_t stream) {
  if (B <= 0 || S <= 0 || window < 0) return -1;
  doc_bounds_kernel<<<B, kBoundsThreads, 0, stream>>>(tokens, S, eos, window == 0 || window > S ? S : window, doc_start, doc_end);
  PB_CHECK_LAUNCH();
  return 0;
}
