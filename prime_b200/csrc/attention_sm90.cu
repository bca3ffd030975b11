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
#include "common.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int BQ = 64;    // forward / dQ query block
constexpr int BKV = 64;   // key block
constexpr int BQB = 32;   // query tile of the dK/dV kernel

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
// D[16x8] += A[16x16] · B[16x8], bf16 in, fp32 accumulate
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}

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
// B operands of two n8 blocks (n0, n0 + 8) for k16 at k0, from a tile stored [n][k] (k contiguous): b[0], b[1] | b[2], b[3]
template <int D>
__device__ __forceinline__ void ld_b_nk(uint32_t base, int n0, int k0, uint32_t (&b)[4]) {
  const int l = threadIdx.x & 31;
  ldsm_x4(base + (uint32_t)((n0 + (l & 7) + (l >> 4) * 8) * Tile<D>::kLd + k0 + ((l >> 3) & 1) * 8) * 2, b);
}
// B operands of two n8 blocks (n0, n0 + 8) for k16 at k0, from a tile stored [k][n] (n contiguous)
template <int D>
__device__ __forceinline__ void ld_b_kn(uint32_t base, int n0, int k0, uint32_t (&b)[4]) {
  const int l = threadIdx.x & 31;
  ldsm_x4_t(base + (uint32_t)((k0 + (l & 7) + ((l >> 3) & 1) * 8) * Tile<D>::kLd + n0 + (l >> 4) * 8) * 2, b);
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

// ------------------------------------------------------------------------------------------------------------------ forward
// kDoc: lower-bounded causal masking. Query q sees key k iff lo[q] <= k <= q (lo = doc_start). lo never decreases along a row,
// so the key loop starts at the tile of lo[q0]; only tiles below lo[q0 + BQ - 1] and the diagonal tile need a mask, the others
// take the plain path.
template <int D, bool kDoc>
__global__ void __launch_bounds__(kThreads) flash_fwd_kernel(const AttnParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int qb = (int)blockIdx.x, bh = (int)blockIdx.y;
  const int b = bh / p.H, h = bh - b * p.H, hk = h / (p.H / p.Hkv);
  const int W = (p.H + 2 * p.Hkv) * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* base = p.qkv + (int64_t)b * p.S * W;
  const uint32_t sq = smem_u32(smem);
  const uint32_t skv = sq + Tile<D>::bytes(BQ);  // [stage][K | V]
  constexpr uint32_t kKV = Tile<D>::bytes(BKV);

  const int q0 = qb * BQ;
  const int n_kv = p.causal ? qb + 1 : p.S / BKV;
  // kDoc: first key tile, document start of the block's last row, document starts of this thread's two rows
  const int* ds = kDoc ? p.doc_start + (int64_t)b * p.S : nullptr;
  const int j0 = kDoc ? ds[q0] / BKV : 0;
  const int ds_max = kDoc ? ds[q0 + BQ - 1] : 0;
  const int rds[2] = {kDoc ? ds[q0 + warp * 16 + g] : 0, kDoc ? ds[q0 + warp * 16 + g + 8] : 0};
  load_tile<D>(sq, base + (int64_t)q0 * W + h * D, W, BQ);
  load_tile<D>(skv, base + (int64_t)j0 * BKV * W + p.H * D + hk * D, W, BKV);
  load_tile<D>(skv + kKV, base + (int64_t)j0 * BKV * W + (p.H + p.Hkv) * D + hk * D, W, BKV);
  cp_async_commit();

  uint32_t qf[D / 16][4];
  float o[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

  for (int j = j0; j < n_kv; ++j) {
    const int st = (j - j0) & 1;
    if (j + 1 < n_kv) {  // prefetch the next key/value tile into the other stage
      const int k1 = (j + 1) * BKV;
      const uint32_t nxt = skv + (st ^ 1) * 2 * kKV;
      load_tile<D>(nxt, base + (int64_t)k1 * W + p.H * D + hk * D, W, BKV);
      load_tile<D>(nxt + kKV, base + (int64_t)k1 * W + (p.H + p.Hkv) * D + hk * D, W, BKV);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    if (j == j0) {
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) ld_a<D>(sq, warp * 16, kk * 16, qf[kk]);
    }
    const uint32_t sk = skv + st * 2 * kKV, sv = sk + kKV;
    float s[BKV / 8][4];
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
      for (int n = 0; n < BKV / 8; n += 2) {
        uint32_t bf[4];
        ld_b_nk<D>(sk, n * 8, kk * 16, bf);
        mma16816(s[n], qf[kk], bf[0], bf[1]);
        mma16816(s[n + 1], qf[kk], bf[2], bf[3]);
      }
    }
    // online softmax (log2 domain); rows g and g + 8 of this warp's 16
    const bool diag = p.causal && j == qb;
    const bool edge = kDoc && (diag || j * BKV < ds_max);
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = s[n][e] * p.scale_log2;
        if constexpr (kDoc) {
          if (edge) {
            const int qi = q0 + warp * 16 + g + (e >> 1) * 8, ki = j * BKV + n * 8 + 2 * t + (e & 1);
            if (ki > qi || ki < rds[e >> 1]) v = -INFINITY;
          }
        } else if (diag) {
          const int qi = warp * 16 + g + (e >> 1) * 8, ki = n * 8 + 2 * t + (e & 1);
          if (ki > qi) v = -INFINITY;
        }
        s[n][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
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
    for (int kk = 0; kk < BKV / 16; ++kk) {
#pragma unroll
      for (int n = 0; n < D / 8; n += 2) {
        uint32_t bf[4];
        ld_b_kn<D>(sv, n * 8, kk * 16, bf);
        mma16816(o[n], pf[kk], bf[0], bf[1]);
        mma16816(o[n + 1], pf[kk], bf[2], bf[3]);
      }
    }
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

// store a 16-row x D fp32 accumulator (mma C layout) as bf16 into rows [row0, row0 + 16) of a [.., ld] buffer at column col0,
// optionally un-rotating the interleaved RoPE pairs (position = sequence index of the row)
template <int D>
__device__ __forceinline__ void store_rows(__nv_bfloat16* dst, int64_t ld, int row0, int s0, float (&acc)[D / 8][4], const AttnParams& p,
                                           bool rope) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + g + r * 8, pos = s0 + g + r * 8;
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

// kDoc: the query-tile loop stops at the tile holding end[b, k0 + BKV - 1] (end never decreases, so no later query sees a key of
// this block) and Pᵀ is zero unless lo[q] <= key <= q; the tile's lo values are staged in shared memory after lse2 and delta.
template <int D, bool kDoc>
__global__ void __launch_bounds__(kThreads) bwd_dkdv_kernel(const AttnParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int kb = (int)blockIdx.x, bhk = (int)blockIdx.y;
  const int b = bhk / p.Hkv, hk = bhk - b * p.Hkv, grp = p.H / p.Hkv;
  const int W = (p.H + 2 * p.Hkv) * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* base = p.qkv + (int64_t)b * p.S * W;
  const __nv_bfloat16* dbase = p.dout + (int64_t)b * p.S * (p.H * D);
  const uint32_t sk = smem_u32(smem), sv = sk + Tile<D>::bytes(BKV);
  const uint32_t sq = sv + Tile<D>::bytes(BKV), sdo = sq + Tile<D>::bytes(BQB);
  float* s_ld = reinterpret_cast<float*>(smem + 2 * Tile<D>::bytes(BKV) + 2 * Tile<D>::bytes(BQB));  // [lse2 BQB | delta BQB]
  int* s_ds = reinterpret_cast<int*>(s_ld + 2 * BQB);  // kDoc: [doc_start BQB]
  const int k0 = kb * BKV;
  load_tile<D>(sk, base + (int64_t)k0 * W + (p.H + hk) * D, W, BKV);
  load_tile<D>(sv, base + (int64_t)k0 * W + (p.H + p.Hkv + hk) * D, W, BKV);
  cp_async_commit();

  float dk[D / 8][4], dv[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[i][e] = dv[i][e] = 0.f;

  const int qt0 = p.causal ? k0 / BQB : 0;
  const int qt_doc = kDoc ? (p.doc_end[(int64_t)b * p.S + k0 + BKV - 1] + BQB - 1) / BQB : 0;
  for (int hh = 0; hh < grp; ++hh) {
    const int h = hk * grp + hh;
    for (int qt = qt0; qt < (kDoc ? qt_doc : p.S / BQB); ++qt) {
      const int q0 = qt * BQB;
      __syncthreads();  // the previous tile has been consumed
      load_tile<D>(sq, base + (int64_t)q0 * W + h * D, W, BQB);
      load_tile<D>(sdo, dbase + (int64_t)q0 * (p.H * D) + h * D, p.H * D, BQB);
      cp_async_commit();
      if (threadIdx.x < BQB) s_ld[threadIdx.x] = p.lse2[((int64_t)b * p.H + h) * p.S + q0 + threadIdx.x];
      else if (threadIdx.x < 2 * BQB) s_ld[threadIdx.x] = p.delta[((int64_t)b * p.H + h) * p.S + q0 + threadIdx.x - BQB];
      if constexpr (kDoc) {
        if (threadIdx.x >= 2 * BQB && threadIdx.x < 3 * BQB) s_ds[threadIdx.x - 2 * BQB] = p.doc_start[(int64_t)b * p.S + q0 + threadIdx.x - 2 * BQB];
      }
      cp_async_wait<0>();
      __syncthreads();
      // Sᵀ = K Qᵀ and dPᵀ = V dOᵀ: 16 keys (this warp) x BQB queries
      float st[BQB / 8][4], dpt[BQB / 8][4];
#pragma unroll
      for (int n = 0; n < BQB / 8; ++n)
#pragma unroll
        for (int e = 0; e < 4; ++e) st[n][e] = dpt[n][e] = 0.f;
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        uint32_t ka[4], va[4];
        ld_a<D>(sk, warp * 16, kk * 16, ka);
        ld_a<D>(sv, warp * 16, kk * 16, va);
#pragma unroll
        for (int n = 0; n < BQB / 8; n += 2) {
          uint32_t bq[4], bo[4];
          ld_b_nk<D>(sq, n * 8, kk * 16, bq);
          ld_b_nk<D>(sdo, n * 8, kk * 16, bo);
          mma16816(st[n], ka, bq[0], bq[1]);
          mma16816(st[n + 1], ka, bq[2], bq[3]);
          mma16816(dpt[n], va, bo[0], bo[1]);
          mma16816(dpt[n + 1], va, bo[2], bo[3]);
        }
      }
      // Pᵀ = exp2(s·scale·log2e − lse2[q]) (0 where q < key), dSᵀ = Pᵀ ∘ (dPᵀ·scale − delta·scale)
      uint32_t pa[BQB / 16][4], da[BQB / 16][4];
#pragma unroll
      for (int n = 0; n < BQB / 8; ++n) {
        float pv[4], dsv[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qi = n * 8 + 2 * t + (e & 1), ki = k0 + warp * 16 + g + (e >> 1) * 8;
          float pe = fast_exp2(st[n][e] * p.scale_log2 - s_ld[qi]);
          if constexpr (kDoc) {
            if (q0 + qi < ki || s_ds[qi] > ki) pe = 0.f;
          } else if (p.causal && q0 + qi < ki) {
            pe = 0.f;
          }
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
#pragma unroll
        for (int n = 0; n < D / 8; n += 2) {
          uint32_t bo[4], bq[4];
          ld_b_kn<D>(sdo, n * 8, kk * 16, bo);
          ld_b_kn<D>(sq, n * 8, kk * 16, bq);
          mma16816(dv[n], pa[kk], bo[0], bo[1]);
          mma16816(dv[n + 1], pa[kk], bo[2], bo[3]);
          mma16816(dk[n], da[kk], bq[0], bq[1]);
          mma16816(dk[n + 1], da[kk], bq[2], bq[3]);
        }
      }
    }
  }
  __nv_bfloat16* dst = p.dqkv + (int64_t)b * p.S * W;
  store_rows<D>(dst + (p.H + hk) * D, W, k0 + warp * 16, k0 + warp * 16, dk, p, p.rope_cos != nullptr);
  store_rows<D>(dst + (p.H + p.Hkv + hk) * D, W, k0 + warp * 16, k0 + warp * 16, dv, p, false);
}

// kDoc: key tiles from lo[b, q0] / BKV to the diagonal, masks as in the forward
template <int D, bool kDoc>
__global__ void __launch_bounds__(kThreads) bwd_dq_kernel(const AttnParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int qb = (int)blockIdx.x, bh = (int)blockIdx.y;
  const int b = bh / p.H, h = bh - b * p.H, hk = h / (p.H / p.Hkv);
  const int W = (p.H + 2 * p.Hkv) * D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* base = p.qkv + (int64_t)b * p.S * W;
  const uint32_t sq = smem_u32(smem), sdo = sq + Tile<D>::bytes(BQ);
  const uint32_t sk = sdo + Tile<D>::bytes(BQ), sv = sk + Tile<D>::bytes(BKV);
  const int q0 = qb * BQ;
  load_tile<D>(sq, base + (int64_t)q0 * W + h * D, W, BQ);
  load_tile<D>(sdo, p.dout + ((int64_t)b * p.S + q0) * (p.H * D) + h * D, p.H * D, BQ);
  cp_async_commit();
  float lse[2], del[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int64_t i = (int64_t)bh * p.S + q0 + warp * 16 + g + r * 8;
    lse[r] = p.lse2[i];
    del[r] = p.delta[i];
  }
  float dq[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
  const int n_kv = p.causal ? qb + 1 : p.S / BKV;
  const int* ds = kDoc ? p.doc_start + (int64_t)b * p.S : nullptr;
  const int j0 = kDoc ? ds[q0] / BKV : 0;
  const int ds_max = kDoc ? ds[q0 + BQ - 1] : 0;
  const int rds[2] = {kDoc ? ds[q0 + warp * 16 + g] : 0, kDoc ? ds[q0 + warp * 16 + g + 8] : 0};
  for (int j = j0; j < n_kv; ++j) {
    const int k0 = j * BKV;
    const bool edge = kDoc && (j == qb || k0 < ds_max);
    __syncthreads();
    load_tile<D>(sk, base + (int64_t)k0 * W + (p.H + hk) * D, W, BKV);
    load_tile<D>(sv, base + (int64_t)k0 * W + (p.H + p.Hkv + hk) * D, W, BKV);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    float s[BKV / 8][4], dp[BKV / 8][4];
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[n][e] = dp[n][e] = 0.f;
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      uint32_t qa[4], oa[4];
      ld_a<D>(sq, warp * 16, kk * 16, qa);
      ld_a<D>(sdo, warp * 16, kk * 16, oa);
#pragma unroll
      for (int n = 0; n < BKV / 8; n += 2) {
        uint32_t bk[4], bv[4];
        ld_b_nk<D>(sk, n * 8, kk * 16, bk);
        ld_b_nk<D>(sv, n * 8, kk * 16, bv);
        mma16816(s[n], qa, bk[0], bk[1]);
        mma16816(s[n + 1], qa, bk[2], bk[3]);
        mma16816(dp[n], oa, bv[0], bv[1]);
        mma16816(dp[n + 1], oa, bv[2], bv[3]);
      }
    }
    uint32_t da[BKV / 16][4];
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
      float dsv[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = e >> 1, qi = q0 + warp * 16 + g + r * 8, ki = k0 + n * 8 + 2 * t + (e & 1);
        float pe = fast_exp2(s[n][e] * p.scale_log2 - lse[r]);
        if constexpr (kDoc) {
          if (edge && (ki > qi || ki < rds[r])) pe = 0.f;
        } else if (p.causal && ki > qi) {
          pe = 0.f;
        }
        dsv[e] = pe * (dp[n][e] * p.scale - del[r]);
      }
      da[n >> 1][(n & 1) * 2] = pack_bf16(dsv[0], dsv[1]);
      da[n >> 1][(n & 1) * 2 + 1] = pack_bf16(dsv[2], dsv[3]);
    }
    // dQ += dS K  (k = keys)
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
#pragma unroll
      for (int n = 0; n < D / 8; n += 2) {
        uint32_t bk[4];
        ld_b_kn<D>(sk, n * 8, kk * 16, bk);
        mma16816(dq[n], da[kk], bk[0], bk[1]);
        mma16816(dq[n + 1], da[kk], bk[2], bk[3]);
      }
    }
  }
  store_rows<D>(p.dqkv + (int64_t)b * p.S * W + h * D, W, q0 + warp * 16, q0 + warp * 16, dq, p, p.rope_cos != nullptr);
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
  AttnParams p{(const __nv_bfloat16*)qkv, (__nv_bfloat16*)out, nullptr, nullptr, nullptr, nullptr, lse2,
               B, S, H, Hkv, scale, scale * 1.4426950408889634f, causal, nullptr, nullptr, doc_start, nullptr};
  if (doc_start != nullptr) {
    if (D == 128) return launch_fwd<128, true>(p, stream);
    if (D == 64) return launch_fwd<64, true>(p, stream);
    return -2;
  }
  if (D == 128) return launch_fwd<128, false>(p, stream);
  if (D == 64) return launch_fwd<64, false>(p, stream);
  return -2;
}

// delta: [B, H, S] fp32 scratch.  dqkv: [B, S, (H+2Hkv)·D] bf16, fully overwritten.
// doc_start / doc_end: both null, or both the forward's lower bound and its matching upper bound (causal != 0).
// rope_cos / rope_sin: null, or the fp32 [S, D/2] tables of a forward rotation, whose inverse is fused into the dQ / dK stores.
PB_EXPORT int pb_flash_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse2, float* delta, void* dqkv,
                                const int* doc_start, const int* doc_end, int B, int S, int H, int Hkv, int D, float scale, int causal,
                                const float* rope_cos, const float* rope_sin, cudaStream_t stream) {
  if (S % 128 != 0 || H % Hkv != 0 || (doc_start == nullptr) != (doc_end == nullptr) || (doc_start != nullptr && !causal)) return -1;
  AttnParams p{(const __nv_bfloat16*)qkv, (__nv_bfloat16*)out, (const __nv_bfloat16*)dout, (__nv_bfloat16*)dqkv, lse2, delta, nullptr,
               B, S, H, Hkv, scale, scale * 1.4426950408889634f, causal, rope_cos, rope_sin, doc_start, doc_end};
  if (doc_start != nullptr) {
    if (D == 128) return launch_bwd<128, true>(p, stream);
    if (D == 64) return launch_bwd<64, true>(p, stream);
    return -2;
  }
  if (D == 128) return launch_bwd<128, false>(p, stream);
  if (D == 64) return launch_bwd<64, false>(p, stream);
  return -2;
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
