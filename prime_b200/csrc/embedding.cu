// Token embedding for the sharded engine: forward = row gather straight out of the (possibly peer-resident) parameter shards,
// backward = DETERMINISTIC scatter-add into the fp32 main_grad (sort by token, then one owner per token row — no atomics).
//
//   forward   out[t, :] = W[tok[t], :]         W is sharded by rows over the FSDP group (ZeRO-3): row v lives on rank v / rpr at
//                                              local row v % rpr. The kernel reads the owner's shard through its NVLink mapping —
//                                              only the rows a micro-batch actually uses cross the link ("all-gather ⊕ lookup");
//                                              with an unsharded table n = 1 and this is a plain local gather.
//   backward  main_grad[v, :] += Σ_{t: tok[t]=v} dOut[t, :]   in ascending t order for every v (bitwise reproducible).
//             kernel 1 sorts (token, position) keys with a shared-memory bitonic network (one CTA, <= 16384 keys per launch; longer
//             inputs are processed chunk by chunk in stream order, which keeps the sum order fixed);
//             kernel 2 gives every run of equal tokens to exactly one CTA column-slice, which walks the run in order.
//
// Replaces torch's embedding / embedding_dense_backward (radix sort + atomics, ~1 % of the Llama-1B step in round 1).
#include "common.cuh"

using namespace pb;

namespace {

constexpr int kMaxPeers = 8;
struct PeerPtrs {
  void* p[kMaxPeers];
  int n;
};

__global__ void __launch_bounds__(256) embedding_fwd_kernel(const int64_t* __restrict__ tokens, int64_t T, PeerPtrs w, int rpr, int dim,
                                                            __nv_bfloat16* __restrict__ out) {
  const int vec = dim >> 3;  // 16-byte vectors per row
  const int64_t total = T * vec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / vec;
    const int c = (int)(i - t * vec);
    const int64_t v = tokens[t];
    const int owner = (int)(v / rpr);
    const int64_t lr = v - (int64_t)owner * rpr;
    const bf16x8* src = reinterpret_cast<const bf16x8*>(reinterpret_cast<const __nv_bfloat16*>(w.p[owner]) + lr * dim) + c;
    // shards are written by the optimizer kernels of a PREVIOUS step (flag barrier in between) and are read-only now: the
    // non-coherent streaming path is safe for peer memory too (L1 is invalidated at every kernel boundary)
    stg_stream(reinterpret_cast<bf16x8*>(out + t * dim) + c, ldg_stream(src));
  }
}

// ---------------------------------------------------------------------------------------------- backward, kernel 1: sort
__global__ void __launch_bounds__(1024) embedding_sort_kernel(const int64_t* __restrict__ tokens, int n, int n_pad, int pos0,
                                                              unsigned long long* __restrict__ sorted) {
  extern __shared__ unsigned long long keys[];
  for (int i = threadIdx.x; i < n_pad; i += blockDim.x)
    keys[i] = i < n ? (((unsigned long long)tokens[i] << 32) | (unsigned)(pos0 + i)) : ~0ull;
  __syncthreads();
  for (int k = 2; k <= n_pad; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n_pad; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = keys[i], b = keys[l];
          const bool up = (i & k) == 0;
          if ((a > b) == up) {
            keys[i] = b;
            keys[l] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) sorted[i] = keys[i];
}

// ---------------------------------------------------------------------------------------------- backward, kernel 2: segmented sum
// grid.x: ranges of `kRange` consecutive sorted entries; grid.y: 1024-column slices. A run of equal tokens belongs to the CTA whose
// range contains the run's first entry; that CTA follows the run past the end of its range.
constexpr int kRange = 16;

__global__ void __launch_bounds__(128) embedding_bwd_kernel(const unsigned long long* __restrict__ sorted, int n,
                                                            const __nv_bfloat16* __restrict__ dout, float* __restrict__ grad, int dim) {
  const int col = (blockIdx.y * 128 + threadIdx.x) * 8;
  if (col >= dim) return;
  const int start = blockIdx.x * kRange, end = min(n, start + kRange);
  int i = start;
  if (i > 0) {
    const unsigned prev = (unsigned)(sorted[i - 1] >> 32);
    while (i < end && (unsigned)(sorted[i] >> 32) == prev) ++i;  // tail of a run owned by an earlier CTA
  }
  while (i < end) {
    const unsigned tok = (unsigned)(sorted[i] >> 32);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int j = i;
    do {
      const unsigned pos = (unsigned)(sorted[j] & 0xffffffffull);
      float f[8];
      unpack8(ldg_stream(reinterpret_cast<const bf16x8*>(dout + (int64_t)pos * dim + col)), f);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += f[k];
      ++j;
    } while (j < n && (unsigned)(sorted[j] >> 32) == tok);
    float4* g = reinterpret_cast<float4*>(grad + (int64_t)tok * dim + col);
    float4 g0 = g[0], g1 = g[1];
    g0.x += acc[0], g0.y += acc[1], g0.z += acc[2], g0.w += acc[3];
    g1.x += acc[4], g1.y += acc[5], g1.z += acc[6], g1.w += acc[7];
    g[0] = g0;
    g[1] = g1;
    i = j;
  }
}

// ---------------------------------------------------------------------------------------------- all-gather by peer loads (copy)
// dst[r * n_per_rank + i] = src.p[r][i]: explicit gather of a row-sharded parameter (small-M fallback of pb_gemm_wgather, tests,
// checkpoint export). 16-byte vectors.
__global__ void __launch_bounds__(512) allgather_copy_kernel(PeerPtrs src, int64_t nvec_per_rank, uint4* __restrict__ dst) {
  const int64_t total = nvec_per_rank * src.n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / nvec_per_rank);
    const int64_t k = i - (int64_t)r * nvec_per_rank;
    dst[i] = ld_relaxed_sys_u4(reinterpret_cast<const uint4*>(src.p[r]) + k);
  }
}

}  // namespace

PB_EXPORT int pb_embedding_fwd(const int64_t* tokens, int64_t T, const PeerPtrs* w, int rows_per_rank, int dim, void* out,
                               cudaStream_t stream) {
  if (dim % 8 != 0 || w->n < 1 || w->n > kMaxPeers || rows_per_rank <= 0) return -1;
  if (T == 0) return 0;
  const int64_t total = T * (dim >> 3);
  int64_t grid = (total + 255) / 256;
  if (grid > 132 * 16) grid = 132 * 16;
  embedding_fwd_kernel<<<(unsigned)grid, 256, 0, stream>>>(tokens, T, *w, rows_per_rank, dim, reinterpret_cast<__nv_bfloat16*>(out));
  PB_CHECK_LAUNCH();
  return 0;
}

// Step 1 (can run as soon as the token ids exist, e.g. on a side stream during the FORWARD pass — it is one CTA for ~0.2 ms):
// sorted[pos0 .. pos0+n) = (token << 32 | position) keys of every 16384-token chunk, ascending.
PB_EXPORT int pb_embedding_sort(const int64_t* tokens, int64_t T, unsigned long long* sorted, cudaStream_t stream) {
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(embedding_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 8);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  for (int64_t pos0 = 0; pos0 < T; pos0 += 16384) {
    const int n = (int)((T - pos0) < 16384 ? (T - pos0) : 16384);
    int n_pad = 2;
    while (n_pad < n) n_pad <<= 1;
    embedding_sort_kernel<<<1, 1024, (size_t)n_pad * 8, stream>>>(tokens + pos0, n, n_pad, (int)pos0, sorted + pos0);
    PB_CHECK_LAUNCH();
  }
  return 0;
}

// Step 2: grad [V, dim] fp32 += segmented sums of dout rows, chunk after chunk in stream order (fixed summation order).
PB_EXPORT int pb_embedding_scatter(const unsigned long long* sorted, int64_t T, const void* dout, float* grad, int dim, cudaStream_t stream) {
  if (dim % 8 != 0) return -1;
  for (int64_t pos0 = 0; pos0 < T; pos0 += 16384) {
    const int n = (int)((T - pos0) < 16384 ? (T - pos0) : 16384);
    dim3 grid((n + kRange - 1) / kRange, (dim + 1023) / 1024);
    embedding_bwd_kernel<<<grid, 128, 0, stream>>>(sorted + pos0, n, reinterpret_cast<const __nv_bfloat16*>(dout), grad, dim);
    PB_CHECK_LAUNCH();
  }
  return 0;
}

PB_EXPORT int pb_allgather_copy(const PeerPtrs* src, int64_t bytes_per_rank, void* dst, cudaStream_t stream) {
  if (bytes_per_rank % 16 != 0 || src->n < 1 || src->n > kMaxPeers) return -1;
  if (bytes_per_rank == 0) return 0;
  allgather_copy_kernel<<<132 * 4, 512, 0, stream>>>(*src, bytes_per_rank / 16, reinterpret_cast<uint4*>(dst));
  PB_CHECK_LAUNCH();
  return 0;
}
