// Memory-bound Llama block ops for sm_90a: RMSNorm (+fused residual add), RoPE,
// SwiGLU, fused softmax-cross-entropy (forward + in-place gradient).
// All kernels: 16-byte vector accesses, fp32 math, bf16 storage, one pass over HBM
// wherever the op allows it.  Roofline target: measured copy bandwidth (MEASURED_PEAKS.json).
#include "common.cuh"

using namespace pb;

// --------------------------------------------------------------------------------------
// RMSNorm forward:  h = x (+ res);  y = h * rstd(h) * w
// one CTA per row; each thread keeps its slice of the row in registers (single HBM read).
// --------------------------------------------------------------------------------------
template <int MAXV, bool HAS_RES>
__global__ void __launch_bounds__(256) rmsnorm_fwd_kernel(const bf16x8* __restrict__ x, const bf16x8* __restrict__ res,
                                                          const bf16x8* __restrict__ w, bf16x8* __restrict__ y,
                                                          bf16x8* __restrict__ h_out, float* __restrict__ rstd_out,
                                                          int nvec, float inv_d, float eps) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const bf16x8* xr = x + row * nvec;
  float vals[MAXV][8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = threadIdx.x + i * blockDim.x;
    if (c < nvec) {
      unpack8(ldg_stream(xr + c), vals[i]);
      if (HAS_RES) {
        float r[8];
        unpack8(ldg_stream(res + row * nvec + c), r);
#pragma unroll
        for (int j = 0; j < 8; ++j) vals[i][j] += r[j];
        // round-trip through bf16 so the normalised value matches what is stored as h
        bf16x8 hp = pack8(vals[i]);
        h_out[row * nvec + c] = hp;
        unpack8(hp, vals[i]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += vals[i][j] * vals[i][j];
    }
  }
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss * inv_d + eps);
  if (threadIdx.x == 0) rstd_out[row] = rstd;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = threadIdx.x + i * blockDim.x;
    if (c < nvec) {
      float wv[8];
      unpack8(w[c], wv);
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = vals[i][j] * rstd * wv[j];
      stg_stream(y + row * nvec + c, pack8(o));
    }
  }
}

PB_EXPORT int pb_rmsnorm_fwd(const void* x, const void* res, const void* w, void* y, void* h_out, float* rstd, int64_t R,
                             int D, float eps, cudaStream_t stream) {
  if (D % 8 != 0 || D > 256 * 8 * 8) return -1;
  const int nvec = D / 8;
  int threads = ((nvec + 31) / 32) * 32;
  if (threads > 256) threads = 256;
  const int vpt = (nvec + threads - 1) / threads;
#define LAUNCH(MV)                                                                                                   \
  if (res)                                                                                                           \
    rmsnorm_fwd_kernel<MV, true><<<(unsigned)R, threads, 0, stream>>>((const bf16x8*)x, (const bf16x8*)res,          \
                                                                      (const bf16x8*)w, (bf16x8*)y, (bf16x8*)h_out,  \
                                                                      rstd, nvec, 1.f / D, eps);                     \
  else                                                                                                               \
    rmsnorm_fwd_kernel<MV, false><<<(unsigned)R, threads, 0, stream>>>((const bf16x8*)x, nullptr, (const bf16x8*)w,  \
                                                                       (bf16x8*)y, nullptr, rstd, nvec, 1.f / D, eps);
  if (vpt <= 1) { LAUNCH(1) } else if (vpt <= 2) { LAUNCH(2) } else if (vpt <= 4) { LAUNCH(4) } else { LAUNCH(8) }
#undef LAUNCH
  PB_CHECK_LAUNCH();
  return 0;
}

// --------------------------------------------------------------------------------------
// RMSNorm backward.
//   g = dy * w ; dx = rstd * (g - h * rstd^2 * mean(g*h)) (+ dres) ; dw += sum_rows(dy * h * rstd)
// Persistent CTAs stride over rows and keep per-column dw partials in registers; a second
// kernel folds the [grid, D] partials (deterministic order) into the fp32 weight gradient.
// --------------------------------------------------------------------------------------
template <int MAXV, bool HAS_DRES>
__global__ void __launch_bounds__(256, MAXV == 1 ? 4 : 1) rmsnorm_bwd_kernel(const bf16x8* __restrict__ dy, const bf16x8* __restrict__ h,
                                                          const bf16x8* __restrict__ w, const float* __restrict__ rstd,
                                                          const bf16x8* __restrict__ dres, bf16x8* __restrict__ dx,
                                                          float* __restrict__ dw_partial, int64_t R, int nvec,
                                                          float inv_d) {
  __shared__ float red[32];
  float wv[MAXV][8], dwacc[MAXV][8];
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = threadIdx.x + i * blockDim.x;
#pragma unroll
    for (int j = 0; j < 8; ++j) dwacc[i][j] = 0.f;
    if (c < nvec) unpack8(w[c], wv[i]);
  }
  // Software pipeline over rows: the raw 16-byte loads of the NEXT row are issued before the block reduction of the current one,
  // so the ≈1 µs HBM latency hides behind reduce + normalise + store instead of being paid once per row per CTA.
  bf16x8 nd[MAXV], nh[MAXV], nr[MAXV];
  auto fetch = [&](int64_t row) {
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int c = threadIdx.x + i * blockDim.x;
      if (c < nvec) {
        nd[i] = ldg_stream(dy + row * nvec + c);
        nh[i] = ldg_stream(h + row * nvec + c);
        if (HAS_DRES) nr[i] = ldg_stream(dres + row * nvec + c);
      }
    }
  };
  if ((int64_t)blockIdx.x < R) fetch(blockIdx.x);
  for (int64_t row = blockIdx.x; row < R; row += gridDim.x) {
    float g[MAXV][8], hv[MAXV][8], rv[MAXV][8];
    const float rs = rstd[row];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int c = threadIdx.x + i * blockDim.x;
      if (c < nvec) {
        float d[8];
        unpack8(nd[i], d);
        unpack8(nh[i], hv[i]);
        if (HAS_DRES) unpack8(nr[i], rv[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          g[i][j] = d[j] * wv[i][j];
          dot += g[i][j] * hv[i][j];
          dwacc[i][j] += d[j] * hv[i][j] * rs;
        }
      }
    }
    if (row + gridDim.x < R) fetch(row + gridDim.x);  // in flight during the reduction and the stores below
    dot = block_sum(dot, red);
    const float coef = dot * inv_d * rs * rs * rs;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      const int c = threadIdx.x + i * blockDim.x;
      if (c < nvec) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = g[i][j] * rs - hv[i][j] * coef;
        if (HAS_DRES) {
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += rv[i][j];
        }
        stg_stream(dx + row * nvec + c, pack8(o));
      }
    }
  }
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = threadIdx.x + i * blockDim.x;
    if (c < nvec) {
      float4* dst = reinterpret_cast<float4*>(dw_partial + (int64_t)blockIdx.x * nvec * 8 + c * 8);
      dst[0] = make_float4(dwacc[i][0], dwacc[i][1], dwacc[i][2], dwacc[i][3]);
      dst[1] = make_float4(dwacc[i][4], dwacc[i][5], dwacc[i][6], dwacc[i][7]);
    }
  }
}

// 32 columns x 8 row-lanes per CTA: coalesced 128 B row segments, 8-way parallel over the partial rows.
__global__ void __launch_bounds__(256) colsum_partials_kernel(const float* __restrict__ partial, float* __restrict__ out,
                                                              int nparts, int D, int accumulate) {
  __shared__ float sm[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  float s = 0.f;
  if (c < D)
    for (int p = ty; p < nparts; p += 8) s += partial[(int64_t)p * D + c];
  sm[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && c < D) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sm[k][tx];
    out[c] = accumulate ? out[c] + t : t;
  }
}

// dw_partial must hold grid*D floats; `grid_out` reports the grid used (query with R<0).
PB_EXPORT int pb_rmsnorm_bwd_grid(int64_t R) {
  // 4 resident CTAs per SM (register-capped by __launch_bounds__): each row iteration is load → block reduction → store, i.e. latency-bound per CTA, so HBM is only
  // saturated by many CTAs in flight (2 per SM measured 28 % of copy bandwidth). Cost: a [grid, D] fp32 partial buffer.
  int64_t g = 132 * 4;
  return (int)(R < g ? R : g);
}

PB_EXPORT int pb_rmsnorm_bwd(const void* dy, const void* h, const void* w, const float* rstd, const void* dres, void* dx,
                             float* dw_partial, float* dw, int dw_accumulate, int64_t R, int D, cudaStream_t stream) {
  if (D % 8 != 0 || D > 256 * 8 * 8) return -1;
  const int nvec = D / 8;
  int threads = ((nvec + 31) / 32) * 32;
  if (threads > 256) threads = 256;
  const int vpt = (nvec + threads - 1) / threads;
  const int grid = pb_rmsnorm_bwd_grid(R);
#define LAUNCH(MV)                                                                                                     \
  if (dres)                                                                                                            \
    rmsnorm_bwd_kernel<MV, true><<<grid, threads, 0, stream>>>((const bf16x8*)dy, (const bf16x8*)h, (const bf16x8*)w,  \
                                                               rstd, (const bf16x8*)dres, (bf16x8*)dx, dw_partial, R,  \
                                                               nvec, 1.f / D);                                         \
  else                                                                                                                 \
    rmsnorm_bwd_kernel<MV, false><<<grid, threads, 0, stream>>>((const bf16x8*)dy, (const bf16x8*)h, (const bf16x8*)w, \
                                                                rstd, nullptr, (bf16x8*)dx, dw_partial, R, nvec,       \
                                                                1.f / D);
  if (vpt <= 1) { LAUNCH(1) } else if (vpt <= 2) { LAUNCH(2) } else if (vpt <= 4) { LAUNCH(4) } else { LAUNCH(8) }
#undef LAUNCH
  PB_CHECK_LAUNCH();
  colsum_partials_kernel<<<(D + 31) / 32, 256, 0, stream>>>(dw_partial, dw, grid, D, dw_accumulate);
  PB_CHECK_LAUNCH();
  return 0;
}

// --------------------------------------------------------------------------------------
// RoPE, in place on the fused QKV activation [tokens, total_heads, D]; the first
// `rot_heads` heads (all of Q then all of K) are rotated, V is left alone.
// Interleaved-pair convention; cos/sin fp32 [S, D/2].  sign=-1 gives the backward pass.
// --------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rope_inplace_kernel(bf16x8* __restrict__ qkv, const float4* __restrict__ cosb,
                                                           const float4* __restrict__ sinb, int64_t tokens, int S,
                                                           int rot_heads, int total_heads, int vec_per_head, float sign) {
  const int64_t per_tok = (int64_t)rot_heads * vec_per_head;
  const int64_t total = tokens * per_tok;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t tok = i / per_tok;
    const int rem = (int)(i - tok * per_tok);
    const int head = rem / vec_per_head, vh = rem - head * vec_per_head;
    const int pos = (int)(tok % S);
    bf16x8* p = qkv + (tok * total_heads + head) * vec_per_head + vh;
    float v[8];
    unpack8(*p, v);
    const float4 c = cosb[(int64_t)pos * vec_per_head + vh];
    const float4 s = sinb[(int64_t)pos * vec_per_head + vh];
    const float cc[4] = {c.x, c.y, c.z, c.w}, sn[4] = {s.x * sign, s.y * sign, s.z * sign, s.w * sign};
    float o[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      o[2 * j] = v[2 * j] * cc[j] - v[2 * j + 1] * sn[j];
      o[2 * j + 1] = v[2 * j] * sn[j] + v[2 * j + 1] * cc[j];
    }
    *p = pack8(o);
  }
}

PB_EXPORT int pb_rope_inplace(void* qkv, const float* cosb, const float* sinb, int64_t tokens, int S, int rot_heads,
                              int total_heads, int D, float sign, cudaStream_t stream) {
  if (D % 8 != 0) return -1;
  const int64_t total = tokens * rot_heads * (D / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  rope_inplace_kernel<<<(unsigned)blocks, 256, 0, stream>>>((bf16x8*)qkv, (const float4*)cosb, (const float4*)sinb,
                                                           tokens, S, rot_heads, total_heads, D / 8, sign);
  PB_CHECK_LAUNCH();
  return 0;
}

// --------------------------------------------------------------------------------------
// SwiGLU: gate_up [R, 2F] (gate | up) -> out [R, F] = silu(gate) * up ; and its backward.
// --------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) swiglu_fwd_kernel(const bf16x8* __restrict__ gu, bf16x8* __restrict__ out,
                                                         int64_t R, int fvec) {
  const int64_t total = R * fvec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / fvec;
    const int c = (int)(i - r * fvec);
    float g[8], u[8], o[8];
    unpack8(ldg_stream(gu + r * 2 * fvec + c), g);
    unpack8(ldg_stream(gu + r * 2 * fvec + fvec + c), u);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = g[j] / (1.f + __expf(-g[j])) * u[j];
    stg_stream(out + i, pack8(o));
  }
}

__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const bf16x8* __restrict__ gu, const bf16x8* __restrict__ dout,
                                                         bf16x8* __restrict__ dgu, int64_t R, int fvec) {
  const int64_t total = R * fvec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / fvec;
    const int c = (int)(i - r * fvec);
    float g[8], u[8], d[8], dg[8], du[8];
    unpack8(ldg_stream(gu + r * 2 * fvec + c), g);
    unpack8(ldg_stream(gu + r * 2 * fvec + fvec + c), u);
    unpack8(ldg_stream(dout + i), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-g[j]));
      const float silu = g[j] * sg;
      du[j] = d[j] * silu;
      dg[j] = d[j] * u[j] * (sg + silu * (1.f - sg));
    }
    stg_stream(dgu + r * 2 * fvec + c, pack8(dg));
    stg_stream(dgu + r * 2 * fvec + fvec + c, pack8(du));
  }
}

PB_EXPORT int pb_swiglu_fwd(const void* gu, void* out, int64_t R, int F, cudaStream_t stream) {
  if (F % 8 != 0) return -1;
  int64_t blocks = (R * (F / 8) + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  swiglu_fwd_kernel<<<(unsigned)blocks, 256, 0, stream>>>((const bf16x8*)gu, (bf16x8*)out, R, F / 8);
  PB_CHECK_LAUNCH();
  return 0;
}
PB_EXPORT int pb_swiglu_bwd(const void* gu, const void* dout, void* dgu, int64_t R, int F, cudaStream_t stream) {
  if (F % 8 != 0) return -1;
  int64_t blocks = (R * (F / 8) + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  swiglu_bwd_kernel<<<(unsigned)blocks, 256, 0, stream>>>((const bf16x8*)gu, (const bf16x8*)dout, (bf16x8*)dgu, R,
                                                         F / 8);
  PB_CHECK_LAUNCH();
  return 0;
}

// --------------------------------------------------------------------------------------
// Fused softmax cross-entropy: per row, loss = logsumexp(z) - z[target]; the logits buffer is
// overwritten with dloss/dz * scale  (scale = grad multiplier / number of valid targets, read
// from device memory so no host sync is needed).  One CTA per row, two passes (2nd hits L2).
// --------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) cross_entropy_kernel(bf16x8* __restrict__ logits, const int64_t* __restrict__ targets,
                                                            float* __restrict__ losses, const float* __restrict__ scale_ptr,
                                                            int V, int64_t ignore_index) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const int nvec = V / 8;
  bf16x8* zr = logits + row * nvec;
  const int64_t tgt = targets[row];
  float m = -INFINITY, s = 0.f;
  for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
    float z[8];
    unpack8(zr[c], z);
    float lm = z[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) lm = fmaxf(lm, z[j]);
    const float nm = fmaxf(m, lm);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += __expf(z[j] - nm);
    s = s * __expf(m - nm) + acc;
    m = nm;
  }
  const float gm = block_max(m, red);
  s = (m == -INFINITY) ? 0.f : s * __expf(m - gm);
  const float gs = block_sum(s, red);
  const float lse = gm + __logf(gs);
  const bool valid = (tgt != ignore_index);
  const float scale = valid ? *scale_ptr : 0.f;
  if (threadIdx.x == 0) {
    float zt = 0.f;
    if (valid) zt = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(zr)[tgt]);
    losses[row] = valid ? (lse - zt) : 0.f;
  }
  __syncthreads();  // target logit read before anyone overwrites it
  const float inv = 1.f / gs;
  for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
    float z[8], o[8];
    unpack8(zr[c], z);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p = __expf(z[j] - gm) * inv;
      if ((int64_t)(c * 8 + j) == tgt) p -= 1.f;
      o[j] = p * scale;
    }
    zr[c] = pack8(o);
  }
}

// Register-resident variant: every thread keeps its share of the row (VPT 16-byte vectors, all loads issued up front) in registers,
// so the logits are read from memory exactly once and the loads of a row are all in flight together (round 1: one load per loop
// iteration, 0.59 of the HBM roof). The first cut of this kernel was ISSUE-bound (ncu: sm 79 %, dram 39 %): two MUFU.EX2 per element
// (16/clk/SM → 0.23 ms of MUFU alone for a 16384 x 32000 tile) and 64-bit target-index compares per element. Now:
//   pass 1  row max on packed bf16x2 (HMNMX2: one instruction per two logits)
//   pass 2  e = exp2(z·log2e − max·log2e): one FFMA + one MUFU per element, summed in fp32, and written BACK into the registers as
//           bf16 (p ∈ (0, 1]); the target logit is picked by ONE range check per vector
//   pass 3  p·(scale/sum) from the stored e — no second exponential; the target's −1 is patched in by the one thread that owns it
template <int VPT, int THREADS>
__global__ void __launch_bounds__(THREADS) cross_entropy_reg_kernel(bf16x8* __restrict__ logits, const int64_t* __restrict__ targets,
                                                                    float* __restrict__ losses, const float* __restrict__ scale_ptr,
                                                                    int V, int64_t ignore_index) {
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const int nvec = V / 8;
  bf16x8* zr = logits + row * nvec;
  const int64_t tgt64 = targets[row];
  const bool valid = (tgt64 != ignore_index);
  const int tgt = valid ? (int)tgt64 : -1;
  bf16x8 v[VPT];
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int c = threadIdx.x + k * THREADS;
    if (c < nvec) v[k] = ldg_stream(zr + c);
  }
  __nv_bfloat162 m2 = __float2bfloat162_rn(-INFINITY);
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int c = threadIdx.x + k * THREADS;
    if (c < nvec) {
#pragma unroll
      for (int j = 0; j < 4; ++j) m2 = __hmax2(m2, v[k].v[j]);
    }
  }
  const float2 mf = __bfloat1622float2(m2);
  const float gm = block_max(fmaxf(mf.x, mf.y), red);
  const float gml2 = gm * 1.4426950408889634f;
  float s = 0.f, zt = 0.f;
  int t_k = -1, t_j = 0;  // which of my registers holds the target (at most one thread of the block)
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int c = threadIdx.x + k * THREADS;
    if (c < nvec) {
      float z[8];
      unpack8(v[k], z);
      const unsigned d = (unsigned)(tgt - c * 8);
      if (d < 8u) {
        t_k = k, t_j = (int)d;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j == (int)d) zt = z[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        z[j] = exp2f(fmaf(z[j], 1.4426950408889634f, -gml2));
        s += z[j];
      }
      v[k] = pack8(z);
    }
  }
  const float gs = block_sum(s, red);
  const float ztg = block_sum(zt, red);  // exactly one thread holds the target logit (0 elsewhere)
  const float scale = valid ? *scale_ptr : 0.f;
  if (threadIdx.x == 0) losses[row] = valid ? (gm + __logf(gs) - ztg) : 0.f;
  const float f = scale / gs;
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int c = threadIdx.x + k * THREADS;
    if (c < nvec) {
      float o[8];
      unpack8(v[k], o);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] *= f;
      if (k == t_k) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j == t_j) o[j] -= scale;
      }
      stg_stream(zr + c, pack8(o));
    }
  }
}

static int launch_cross_entropy(void* logits, const int64_t* targets, float* losses, const float* scale_ptr, int64_t R, int V,
                                int64_t ignore_index, cudaStream_t stream) {
  if (V % 8 != 0) return -1;
  const int nvec = V / 8;
  if (nvec <= 512 * 8)
    cross_entropy_reg_kernel<8, 512><<<(unsigned)R, 512, 0, stream>>>((bf16x8*)logits, targets, losses, scale_ptr, V, ignore_index);
  else  // larger vocabularies (Llama-3: 128256) would spill the register-resident row: two-pass kernel

    cross_entropy_kernel<<<(unsigned)R, 512, 0, stream>>>((bf16x8*)logits, targets, losses, scale_ptr, V, ignore_index);
  PB_CHECK_LAUNCH();
  return 0;
}

// Whole loss node without a single framework kernel: count the valid targets → gradient scale; the row kernel; a fixed-order sum
// of the per-row losses → mean loss (deterministic). work: >= 2 floats of scratch ([0] = grad_scale / n_valid, [1] = 1 / n_valid).
__global__ void __launch_bounds__(1024) ce_count_kernel(const int64_t* __restrict__ targets, int64_t R, int64_t ignore_index,
                                                        float grad_scale, float* __restrict__ work) {
  __shared__ float red[32];
  float n = 0.f;
  for (int64_t i = threadIdx.x; i < R; i += blockDim.x) n += targets[i] != ignore_index ? 1.f : 0.f;
  n = block_sum(n, red);
  if (threadIdx.x == 0) {
    const float inv = 1.f / fmaxf(n, 1.f);
    work[0] = grad_scale * inv;
    work[1] = inv;
  }
}
__global__ void __launch_bounds__(1024) ce_finalize_kernel(const float* __restrict__ losses, int64_t R, const float* __restrict__ work,
                                                           float* __restrict__ loss_out, float* __restrict__ loss_acc) {
  __shared__ float red[32];
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < R; i += blockDim.x) s += losses[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float mean = s * work[1];
    *loss_out = mean;
    if (loss_acc != nullptr) *loss_acc += mean;  // running sum over the micro-batches of a step (the trainer's logging value)
  }
}
PB_EXPORT int pb_cross_entropy_loss(void* logits, const int64_t* targets, float* losses, float* work, float* loss_out, float* loss_acc,
                                    int64_t R, int V, int64_t ignore_index, float grad_scale, cudaStream_t stream) {
  ce_count_kernel<<<1, 1024, 0, stream>>>(targets, R, ignore_index, grad_scale, work);
  PB_CHECK_LAUNCH();
  int rc = launch_cross_entropy(logits, targets, losses, work, R, V, ignore_index, stream);
  if (rc) return rc;
  ce_finalize_kernel<<<1, 1024, 0, stream>>>(losses, R, work, loss_out, loss_acc);
  PB_CHECK_LAUNCH();
  return 0;
}
