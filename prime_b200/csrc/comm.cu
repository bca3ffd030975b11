// NVLink/NVSwitch peer-memory layer and the fused collective+compute kernels.
//
//  * symmetric heap: one cudaMalloc per rank, exported with cudaIpc and mapped by every peer, so a
//    kernel can ld/st any peer's buffer at (peer_base + offset) through NVSwitch;
//  * device-side flags (st.release.sys / ld.acquire.sys) for stream-ordered signalling — no host
//    sync, no NCCL launch on the hot path; every spin has a wall-clock bound and reports a timeout
//    through a device error word instead of hanging the GPU;
//  * FSDP inner step:   grad reduce-scatter (peer loads in fixed rank order, or one NVSwitch multicast load) ⊕ scale ⊕
//                       sum-of-squares, then clip ⊕ partitioned AdamW ⊕ bf16 cast ⊕ parameter all-gather (peer stores);
//  * DiLoCo outer step: pseudo-gradient ⊕ int8 block quantise, then peer int8 all-gather ⊕ dequant-sum
//                       ⊕ Nesterov ⊕ parameter write-back/all-gather — one kernel pair;
//  * NVLS (multimem) kernels over the multicast heap of csrc/multicast.cu: flag barrier and in-place all-reduce. They live here
//    because every device-side wait goes through spin_wait_ge, and g_spin_timeout_ns is visible in this translation unit only
//    (the library is built without relocatable device code).
#include "common.cuh"

using namespace pb;

constexpr int kMaxPeers = 8;
// Bound of every device-side wait (default 20 s; elastic jobs lower it so a dead peer is detected within a heartbeat period).
__device__ unsigned long long g_spin_timeout_ns = 20ull * 1000ull * 1000ull * 1000ull;

struct PeerPtrs {
  void* p[kMaxPeers];
  int n;
};

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Spin until *flag >= expect (monotone epochs). Returns false on timeout, or as soon as the error word is non-zero (another
// wait already timed out, or the host's watchdog aborted the step because a peer died: SymmetricHeap.abort()).
// err[0] = 1 timeout / 2 host abort; err[1] = flag address offset that timed out (diagnostic).
__device__ __forceinline__ bool spin_wait_ge(const uint32_t* flag, uint32_t expect, uint32_t* err) {
  if ((int32_t)(ld_acquire_sys_u32(flag) - expect) >= 0) return true;
  const unsigned long long t0 = globaltimer_ns(), limit = g_spin_timeout_ns;
  uint32_t spins = 0;
  while ((int32_t)(ld_acquire_sys_u32(flag) - expect) < 0) {
    __nanosleep(64);
    if ((++spins & 63u) == 0) {
      if (err && *reinterpret_cast<volatile uint32_t*>(err) != 0u) return false;
      if (globaltimer_ns() - t0 > limit) {
        if (err) atomicCAS(err, 0u, 1u);
        return false;
      }
    }
  }
  return true;
}

PB_EXPORT int pb_set_spin_timeout_ms(unsigned long long ms) {
  const unsigned long long ns = ms * 1000000ull;
  return (int)cudaMemcpyToSymbol(g_spin_timeout_ns, &ns, sizeof(ns));
}

// multimem PTX on NVSwitch multicast addresses: a load returns the sum over every GPU's copy, a store lands in every copy.
__device__ __forceinline__ float4 mc_ld_reduce_f32x4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void mc_st_f32x4(float* mc, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
// 8 bf16 per access; the switch accumulates in fp32 (.acc::f32) and rounds once.
__device__ __forceinline__ uint4 mc_ld_reduce_bf16x8(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void mc_st_bf16x8(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void mc_red_release_add_u32(uint32_t* mc, uint32_t v) {
  asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}

// ------------------------------------------------------------------------------------------------
// IPC plumbing (host side)
// ------------------------------------------------------------------------------------------------
PB_EXPORT int pb_ipc_alloc(void** ptr, size_t bytes) {
  cudaError_t e = cudaMalloc(ptr, bytes);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaMemset(*ptr, 0, bytes);
}
PB_EXPORT int pb_ipc_free(void* ptr) { return (int)cudaFree(ptr); }
PB_EXPORT int pb_ipc_handle_size() { return (int)sizeof(cudaIpcMemHandle_t); }
PB_EXPORT int pb_ipc_get_handle(void* ptr, void* handle_out) {
  return (int)cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle_out), ptr);
}
PB_EXPORT int pb_ipc_open_handle(const void* handle, void** ptr_out) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  return (int)cudaIpcOpenMemHandle(ptr_out, h, cudaIpcMemLazyEnablePeerAccess);
}
PB_EXPORT int pb_ipc_close_handle(void* ptr) { return (int)cudaIpcCloseMemHandle(ptr); }
PB_EXPORT int pb_enable_peer_access(int peer_device) {
  int can = 0, cur = 0;
  cudaGetDevice(&cur);
  if (peer_device == cur) return 0;
  cudaDeviceCanAccessPeer(&can, cur, peer_device);
  if (!can) return -2;
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();
    return 0;
  }
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// signal / barrier
// ------------------------------------------------------------------------------------------------
// flags live at the same offset in every rank's heap: slot layout [channel][rank].
__global__ void signal_kernel(PeerPtrs flags, int slot, uint32_t value) {
  if ((int)threadIdx.x < flags.n) {
    __threadfence_system();
    st_release_sys_u32(reinterpret_cast<uint32_t*>(flags.p[threadIdx.x]) + slot, value);
  }
}
PB_EXPORT int pb_signal(const PeerPtrs* flags, int slot, uint32_t value, cudaStream_t stream) {
  signal_kernel<<<1, 32, 0, stream>>>(*flags, slot, value);
  PB_CHECK_LAUNCH();
  return 0;
}

// Full barrier across `flags.n` ranks: publish `epoch` into slot[base + my_idx] on every peer, then wait
// until every slot[base + i] in MY heap reached `epoch`.
__global__ void barrier_kernel(PeerPtrs flags, int base_slot, int my_idx, uint32_t epoch, uint32_t* err) {
  const int t = threadIdx.x;
  if (t < flags.n) {
    __threadfence_system();
    st_release_sys_u32(reinterpret_cast<uint32_t*>(flags.p[t]) + base_slot + my_idx, epoch);
    spin_wait_ge(reinterpret_cast<uint32_t*>(flags.p[my_idx]) + base_slot + t, epoch, err);
  }
}
PB_EXPORT int pb_barrier(const PeerPtrs* flags, int base_slot, int my_idx, uint32_t epoch, uint32_t* err,
                         cudaStream_t stream) {
  barrier_kernel<<<1, 32, 0, stream>>>(*flags, base_slot, my_idx, epoch, err);
  PB_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// FSDP phase 1: reduce-scatter of one gradient bucket, over the segments of a SegTable.
//   out[dst_off[s] + i] = scale * sum_p grads[p][src_off[s] + i]   (p in fixed rank order → bitwise identical across runs)
//   sumsq_partial[blockIdx] += sum_i out[i]^2                      (accumulated over buckets; folded by phase 2)
// A flat bucket's shard is one segment; a row-sharded (ZeRO-3) bucket's is one row block per parameter.
// If wait_flags != nullptr the kernel first waits for flag[slot_base + p] >= expect for every peer p (p < grads.n).
// MC: the gradients come as ONE multicast address and the switch sums the copies (one multimem.ld_reduce per 16 bytes instead of
// P peer loads); its summation order is fixed by the hardware, so the result is deterministic but not bitwise equal to rank order.
// ------------------------------------------------------------------------------------------------
constexpr int kMaxSegs = 16;
struct SegTable {
  int64_t src_off[kMaxSegs], dst_off[kMaxSegs], n[kMaxSegs];
  int nseg;
};

// U = independent 16-byte vectors per thread and iteration: with few peers a thread otherwise has one or two loads in flight and
// the kernel runs at half the memory roof (ncu r2: F = 1 → dram 50 %, warps 49 %); U·F loads are issued before any is consumed.
template <int U, int P, bool MC>
__global__ void __launch_bounds__(512) grad_reduce_kernel(PeerPtrs grads, const float* __restrict__ mc_grads, SegTable segs, float scale,
                                                          float* __restrict__ out, float* __restrict__ sumsq_partial,
                                                          const uint32_t* wait_flags, int slot_base, uint32_t expect, uint32_t* err) {
  __shared__ float red[32];
  if (wait_flags != nullptr) {
    __shared__ int s_fail;
    if (threadIdx.x == 0) s_fail = 0;
    __syncthreads();
    if ((int)threadIdx.x < grads.n && !spin_wait_ge(wait_flags + slot_base + threadIdx.x, expect, err)) s_fail = 1;
    __syncthreads();
    if (s_fail) return;  // a peer never signalled: leave the shard untouched, the host raises on the error word
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  float ss = 0.f;
  for (int s = 0; s < segs.nseg; ++s) {
    const int64_t nvec = segs.n[s] >> 2, src = segs.src_off[s];
    float4* o4 = reinterpret_cast<float4*>(out + segs.dst_off[s]);
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < nvec; i0 += stride * U) {
      float4 v[U][P];  // P = compile-time bound on the number of peers (registers are allocated for P, not for kMaxPeers)
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = i0 + u * stride;
        if constexpr (MC) {
          if (i < nvec) v[u][0] = mc_ld_reduce_f32x4(mc_grads + src + 4 * i);
        } else {
#pragma unroll
          for (int p = 0; p < P; ++p)
            if (p < grads.n && i < nvec)
              v[u][p] = ld_relaxed_sys_f4(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(grads.p[p]) + src) + i);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = i0 + u * stride;
        if (i < nvec) {
          float4 acc = MC ? v[u][0] : make_float4(0.f, 0.f, 0.f, 0.f);
          if constexpr (!MC) {
#pragma unroll
            for (int p = 0; p < P; ++p)
              if (p < grads.n) acc.x += v[u][p].x, acc.y += v[u][p].y, acc.z += v[u][p].z, acc.w += v[u][p].w;  // fixed rank order
          }
          acc.x *= scale, acc.y *= scale, acc.z *= scale, acc.w *= scale;
          o4[i] = acc;
          ss += acc.x * acc.x + acc.y * acc.y + acc.z * acc.z + acc.w * acc.w;
        }
      }
    }
  }
  ss = block_sum(ss, red);
  if (threadIdx.x == 0) sumsq_partial[blockIdx.x] += ss;
}

PB_EXPORT int pb_grad_reduce_grid() { return 132 * 2; }

// grads->n = peers (and flags waited on); mc_grads != nullptr selects the switch-side sum at that multicast address, to which
// src_off is relative as it is to every grads->p[p].
PB_EXPORT int pb_grad_reduce(const PeerPtrs* grads, const float* mc_grads, const SegTable* segs, float scale, float* out,
                             float* sumsq_partial, const uint32_t* wait_flags, int slot_base, uint32_t expect, uint32_t* err, int max_ctas,
                             cudaStream_t stream) {
  if (segs->nseg < 0 || segs->nseg > kMaxSegs) return -1;
  for (int i = 0; i < segs->nseg; ++i)
    if ((segs->n[i] | segs->src_off[i] | segs->dst_off[i]) & 3) return -1;
  int grid = pb_grad_reduce_grid();
  if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;  // leave SMs to the backward pass this runs under
  const auto launch = [&](auto kernel) {
    kernel<<<grid, 512, 0, stream>>>(*grads, mc_grads, *segs, scale, out, sumsq_partial, wait_flags, slot_base, expect, err);
  };
  if (mc_grads != nullptr) launch(grad_reduce_kernel<1, 1, true>);
  else if (grads->n == 1) launch(grad_reduce_kernel<4, 1, false>);
  else if (grads->n == 2) launch(grad_reduce_kernel<4, 2, false>);
  else if (grads->n <= 4) launch(grad_reduce_kernel<2, 4, false>);
  else launch(grad_reduce_kernel<1, 8, false>);
  PB_CHECK_LAUNCH();
  return 0;
}

// Fold this rank's sum-of-squares partials, publish to every peer's norm slot, signal.
__global__ void norm_publish_kernel(float* __restrict__ sumsq_partial, int nparts, PeerPtrs norm_slots, PeerPtrs flags,
                                    int my_idx, int flag_slot, uint32_t epoch) {
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) {
    s += sumsq_partial[i];
    sumsq_partial[i] = 0.f;  // ready for the next step
  }
  s = block_sum(s, red);
  if ((int)threadIdx.x < norm_slots.n) {
    reinterpret_cast<float*>(norm_slots.p[threadIdx.x])[my_idx] = s;
    __threadfence_system();
    st_release_sys_u32(reinterpret_cast<uint32_t*>(flags.p[threadIdx.x]) + flag_slot + my_idx, epoch);
  }
}
PB_EXPORT int pb_norm_publish(float* sumsq_partial, int nparts, const PeerPtrs* norm_slots, const PeerPtrs* flags,
                              int my_idx, int flag_slot, uint32_t epoch, cudaStream_t stream) {
  norm_publish_kernel<<<1, 512, 0, stream>>>(sumsq_partial, nparts, *norm_slots, *flags, my_idx, flag_slot, epoch);
  PB_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// FSDP phase 2: clip ⊕ AdamW on this rank's fp32 master shard ⊕ bf16 cast ⊕ all-gather by peer stores.
// ------------------------------------------------------------------------------------------------
struct AdamArgs {
  float lr, beta1, beta2, eps, weight_decay, bc1, bc2, max_norm;
};

__global__ void __launch_bounds__(512) adamw_push_kernel(float* __restrict__ p32, const float* __restrict__ g32,
                                                         float* __restrict__ m, float* __restrict__ v, int64_t n,
                                                         AdamArgs a, const float* norm_slots, int n_norm,
                                                         const uint32_t* wait_flags, int flag_slot, uint32_t epoch,
                                                         PeerPtrs dst, int64_t dst_off, float* gnorm_out, uint32_t* err,
                                                         __nv_bfloat16* mc_dst) {
  // mc_dst != nullptr: the parameter buffer's NVSwitch MULTICAST address (parallel/multicast.py) — one multimem.st per 16 bytes
  // lands in every rank's copy, so the all-gather leaves this GPU once instead of once per peer (1/F of the outbound bytes)
  __shared__ float s_clip;
  __shared__ int s_fail;
  if (threadIdx.x == 0) {
    float clip = 1.f;
    s_fail = 0;
    if (norm_slots != nullptr) {
      float tot = 0.f;
      for (int i = 0; i < n_norm; ++i) {
        if (wait_flags && !spin_wait_ge(wait_flags + flag_slot + i, epoch, err)) s_fail = 1;
        tot += reinterpret_cast<const volatile float*>(norm_slots)[i];
      }
      const float gn = sqrtf(tot);
      if (gnorm_out && blockIdx.x == 0) *gnorm_out = gn;
      if (a.max_norm > 0.f) clip = fminf(1.f, a.max_norm / (gn + 1e-6f));
    }
    s_clip = clip;
  }
  __syncthreads();
  if (s_fail) return;  // global norm unknown: do not touch the optimizer state (the step is void, the host raises)
  const float clip = s_clip;
  const float step_size = a.lr / a.bc1;
  const float inv_sqrt_bc2 = rsqrtf(a.bc2);
  const float decay = 1.f - a.lr * a.weight_decay;
  const int64_t nvec = n >> 3;  // 8 elements per thread-iteration → one 16-byte bf16 store per peer
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    float out[8];
    // all eight 16-byte loads of the iteration are issued before any is consumed (the kernel runs at 50 % occupancy — 62
    // registers — so memory-level parallelism has to come from within the thread; ncu r2: 56 % of DRAM peak with the loads of the
    // second half issued behind the stores of the first)
    float4 p4[2], g4[2], m4[2], v4[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t j = i * 2 + h;
      p4[h] = reinterpret_cast<const float4*>(p32)[j];
      g4[h] = ldg_stream_f4(reinterpret_cast<const float4*>(g32) + j);
      m4[h] = reinterpret_cast<const float4*>(m)[j];
      v4[h] = reinterpret_cast<const float4*>(v)[j];
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t j = i * 2 + h;
      float4 p = p4[h];
      const float4 g = g4[h];
      float4 mm = m4[h];
      float4 vv = v4[h];
      float* pp = &p.x;
      const float* gp = &g.x;
      float* mp = &mm.x;
      float* vp = &vv.x;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float gk = gp[k] * clip;
        mp[k] = a.beta1 * mp[k] + (1.f - a.beta1) * gk;
        vp[k] = a.beta2 * vp[k] + (1.f - a.beta2) * gk * gk;
        const float denom = sqrtf(vp[k]) * inv_sqrt_bc2 + a.eps;
        pp[k] = pp[k] * decay - step_size * mp[k] / denom;
        out[h * 4 + k] = pp[k];
      }
      reinterpret_cast<float4*>(p32)[j] = p;
      reinterpret_cast<float4*>(m)[j] = mm;
      reinterpret_cast<float4*>(v)[j] = vv;
    }
    const bf16x8 packed = pack8(out);
    if (mc_dst != nullptr) {
      const uint4& r = *reinterpret_cast<const uint4*>(&packed);
      asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(reinterpret_cast<bf16x8*>(mc_dst + dst_off) + i),
                   "r"(r.x), "r"(r.y), "r"(r.z), "r"(r.w)
                   : "memory");
    } else {
#pragma unroll
      for (int q = 0; q < kMaxPeers; ++q)
        if (q < dst.n) stg_v4(reinterpret_cast<bf16x8*>(reinterpret_cast<__nv_bfloat16*>(dst.p[q]) + dst_off) + i, packed);
    }
  }
}

PB_EXPORT int pb_adamw_push(float* p32, const float* g32, float* m, float* v, int64_t n, const AdamArgs* a,
                            const float* norm_slots, int n_norm, const uint32_t* wait_flags, int flag_slot,
                            uint32_t epoch, const PeerPtrs* dst, int64_t dst_off, float* gnorm_out, uint32_t* err,
                            void* mc_dst, cudaStream_t stream) {
  if (n % 8 != 0 || dst_off % 8 != 0) return -1;
  adamw_push_kernel<<<132 * 2, 512, 0, stream>>>(p32, g32, m, v, n, *a, norm_slots, n_norm, wait_flags, flag_slot, epoch,
                                                 *dst, dst_off, gnorm_out, err, reinterpret_cast<__nv_bfloat16*>(mc_dst));
  PB_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// DiLoCo outer step.  Shard space (theta0 / momentum / inner master / int8 payload) is one contiguous index range per rank;
// the bf16 parameter buffer is bucketed, so the write-back position of shard element i is  dst_start[b] + (i - shard_start[b])
// for the bucket b that contains i (tables in device memory, <= a few hundred entries, every boundary a multiple of 1024).
// With that table ONE launch covers every bucket (round 1 launched one kernel per bucket).
//
// Vector widths: 16 elements per thread — int8 payload = one 16-byte load per worker (ld.relaxed.sys.v4: peer data, L2-bypass),
// fp32 state = 4 x float4, bf16 parameters = two 16-byte stores per FSDP peer (round 1: 4-byte int8 loads, 8-byte bf16 stores).
// A 1024-element quantisation block is owned by 64 threads (2 warps); a 256-thread CTA walks 4 blocks per iteration.
// ------------------------------------------------------------------------------------------------
struct OuterArgs {
  float lr, momentum, inv_workers;
  int nesterov;
};
struct BucketTable {
  const int64_t* shard_start;  // [nb + 1] ascending, shard_start[nb] = n
  const int64_t* dst_start;    // [nb] element offset in the bf16 parameter buffer
  int nb;
};

__device__ __forceinline__ int64_t table_dst(const BucketTable& t, int64_t i) {
  int lo = 0, hi = t.nb - 1;
  while (lo < hi) {  // last bucket whose shard_start <= i
    const int mid = (lo + hi + 1) >> 1;
    if (t.shard_start[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  return t.dst_start[lo] + (i - t.shard_start[lo]);
}

__device__ __forceinline__ void dequant16(const uint4& q, float sc, float (&g)[16]) {
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int k = 0; k < 4; ++k) g[j * 4 + k] += (float)(int8_t)((w[j] >> (8 * k)) & 0xffu) * sc;
  }
}

// kernel 1: pseudo-gradient ⊕ symmetric int8 block quantisation.  delta = theta0 - theta; q = rint(delta / (absmax/127)).
__global__ void __launch_bounds__(256) pseudograd_quant_kernel(const float* __restrict__ theta0, const float* __restrict__ theta,
                                                               int8_t* __restrict__ q, float* __restrict__ scales, int64_t n) {
  __shared__ float s_max[8];
  const int grp = threadIdx.x >> 6, t64 = threadIdx.x & 63, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t nblk = n >> 10;
  for (int64_t blk0 = (int64_t)blockIdx.x * 4; blk0 < nblk; blk0 += (int64_t)gridDim.x * 4) {
    const int64_t blk = blk0 + grp;
    const bool on = blk < nblk;
    const int64_t base = blk * 1024 + t64 * 16;
    float d[16];
    float am = 0.f;
    if (on) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 a = ldg_stream_f4(reinterpret_cast<const float4*>(theta0 + base) + j);
        const float4 b = ldg_stream_f4(reinterpret_cast<const float4*>(theta + base) + j);
        d[4 * j] = a.x - b.x, d[4 * j + 1] = a.y - b.y, d[4 * j + 2] = a.z - b.z, d[4 * j + 3] = a.w - b.w;
      }
#pragma unroll
      for (int k = 0; k < 16; ++k) am = fmaxf(am, fabsf(d[k]));
    }
    am = warp_max(am);
    __syncthreads();
    if (lane == 0) s_max[warp] = am;
    __syncthreads();
    am = fmaxf(s_max[grp * 2], s_max[grp * 2 + 1]);
    if (!on) continue;
    const float scale = am / 127.f;
    const float inv = scale > 0.f ? 1.f / scale : 0.f;
    // a subnormal scale (absmax < 127·2^-126) divides instead: its reciprocal can overflow to inf, and 0·inf = NaN would clamp to +127
    const bool divide = scale > 0.f && scale < 0x1p-126f;
    if (t64 == 0) scales[blk] = scale;
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t pk = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float x = d[4 * j + k];
        const int v = (int)fmaxf(-127.f, fminf(127.f, rintf(divide ? x / scale : x * inv)));
        pk |= ((uint32_t)v & 0xffu) << (8 * k);
      }
      w[j] = pk;
    }
    *reinterpret_cast<uint4*>(q + base) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

PB_EXPORT int pb_pseudograd_quant(const float* theta0, const float* theta, int8_t* q, float* scales, int64_t n,
                                  cudaStream_t stream) {
  if (n % 1024 != 0) return -1;
  int64_t ctas = (n / 1024 + 3) / 4;
  if (ctas > 132 * 8) ctas = 132 * 8;
  if (ctas < 1) ctas = 1;
  pseudograd_quant_kernel<<<(unsigned)ctas, 256, 0, stream>>>(theta0, theta, q, scales, n);
  PB_CHECK_LAUNCH();
  return 0;
}

// kernel 2: int8 all-gather by peer loads ⊕ dequantise-sum (fixed worker order → bitwise identical theta0 on every worker)
// ⊕ Nesterov SGD on theta0 ⊕ reset of the inner fp32 master ⊕ bf16 write-back to the FSDP group.
// `qs.p[w]` / `ss.p[w]` = worker w's int8 payload / scales for THIS rank's shard (peer-mapped).
__global__ void __launch_bounds__(256) outer_nesterov_kernel(PeerPtrs qs, PeerPtrs ss, float* __restrict__ theta0,
                                                             float* __restrict__ mom, float* __restrict__ theta, int64_t n,
                                                             OuterArgs a, PeerPtrs dst, BucketTable tab, const uint32_t* err) {
  // a failed flag barrier in front of this kernel (a worker died between the rendezvous and the exchange) leaves the error word
  // set: the peers' payloads are not trustworthy, so nothing is read or updated and the host retries on the re-formed group
  if (err != nullptr && *reinterpret_cast<const volatile uint32_t*>(err) != 0u) return;
  const int grp = threadIdx.x >> 6, t64 = threadIdx.x & 63, lane = threadIdx.x & 31;
  const int64_t nblk = n >> 10;
  for (int64_t blk0 = (int64_t)blockIdx.x * 4; blk0 < nblk; blk0 += (int64_t)gridDim.x * 4) {
    const int64_t blk = blk0 + grp;
    if (blk >= nblk) continue;  // whole warps drop out together (a block is two full warps)
    const int64_t base = blk * 1024 + t64 * 16;
    // Every load of the iteration is issued before the first use. Round 1/2a loaded "scale, shuffle, payload" peer by peer: the
    // shuffle needs the scale, so each peer cost a full NVLink round trip (≈2 µs) before the next peer's loads could even issue —
    // W = 8 ran at 377 GB/s per rank. Now lane w fetches peer w's scale (one instruction for all peers), the W payload loads
    // and the local theta0 / momentum loads follow back to back, and only then are the scales broadcast and consumed.
    float sc_l = 0.f;
    const float* sp = nullptr;
#pragma unroll
    for (int w = 0; w < kMaxPeers; ++w)
      if (lane == w) sp = reinterpret_cast<const float*>(ss.p[w]);  // select chain: a dynamic index would spill the struct to local memory
    if (lane < qs.n) asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(sc_l) : "l"(sp + blk));
    uint4 qv[kMaxPeers];
#pragma unroll
    for (int w = 0; w < kMaxPeers; ++w)
      if (w < qs.n) qv[w] = ld_relaxed_sys_u4(reinterpret_cast<const uint4*>(reinterpret_cast<const int8_t*>(qs.p[w]) + base));
    float4 t0v[4], mmv[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      t0v[j] = reinterpret_cast<const float4*>(theta0 + base)[j];
      mmv[j] = reinterpret_cast<const float4*>(mom + base)[j];
    }
    float g[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) g[k] = 0.f;
#pragma unroll
    for (int w = 0; w < kMaxPeers; ++w) {  // fixed worker order → bitwise identical sums on every worker
      const float sc = __shfl_sync(0xffffffffu, sc_l, w);
      if (w < qs.n) dequant16(qv[w], sc, g);
    }
    float outv[16];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float4 t0 = t0v[j];
      float4 mm = mmv[j];
      float* tp = &t0.x;
      float* mp = &mm.x;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float gk = g[4 * j + k] * a.inv_workers;
        const float mk = a.momentum * mp[k] + gk;
        mp[k] = mk;
        const float upd = a.nesterov ? gk + a.momentum * mk : mk;
        tp[k] = tp[k] - a.lr * upd;
        outv[4 * j + k] = tp[k];
      }
      reinterpret_cast<float4*>(theta0 + base)[j] = t0;
      reinterpret_cast<float4*>(mom + base)[j] = mm;
      reinterpret_cast<float4*>(theta + base)[j] = t0;
    }
    const int64_t d0 = table_dst(tab, base);
    const float lo8[8] = {outv[0], outv[1], outv[2], outv[3], outv[4], outv[5], outv[6], outv[7]};
    const float hi8[8] = {outv[8], outv[9], outv[10], outv[11], outv[12], outv[13], outv[14], outv[15]};
    const bf16x8 plo = pack8(lo8), phi = pack8(hi8);
#pragma unroll
    for (int qd = 0; qd < kMaxPeers; ++qd) {
      if (qd < dst.n) {
        bf16x8* o = reinterpret_cast<bf16x8*>(reinterpret_cast<__nv_bfloat16*>(dst.p[qd]) + d0);
        stg_v4(o, plo);
        stg_v4(o + 1, phi);
      }
    }
  }
}

PB_EXPORT int pb_outer_nesterov(const PeerPtrs* qs, const PeerPtrs* ss, float* theta0, float* mom, float* theta, int64_t n,
                                const OuterArgs* a, const PeerPtrs* dst, const int64_t* shard_start, const int64_t* dst_start,
                                int nb, const uint32_t* err, cudaStream_t stream) {
  if (n % 1024 != 0 || nb < 1) return -1;
  int64_t ctas = (n / 1024 + 3) / 4;
  if (ctas > 132 * 8) ctas = 132 * 8;
  if (ctas < 1) ctas = 1;
  BucketTable tab{shard_start, dst_start, nb};
  outer_nesterov_kernel<<<(unsigned)ctas, 256, 0, stream>>>(*qs, *ss, theta0, mom, theta, n, *a, *dst, tab, err);
  PB_CHECK_LAUNCH();
  return 0;
}

// fp32 (uncompressed) outer path: the workers' inner masters live in the symmetric heap; every worker loads the peers' masters
// directly (16-byte ld.relaxed.sys), forms the averaged pseudo-gradient in fixed worker order, applies Nesterov to theta0, stages
// the new master in `theta_new` (peers are still reading `thetas.p[self]`; the caller copies it back after the closing barrier) and
// pushes the bf16 parameters to the FSDP group.
__global__ void __launch_bounds__(256) outer_nesterov_f32_kernel(PeerPtrs thetas, float* __restrict__ theta0, float* __restrict__ mom,
                                                                 float* __restrict__ theta_new, int64_t n, OuterArgs a, PeerPtrs dst,
                                                                 BucketTable tab, const uint32_t* err) {
  if (err != nullptr && *reinterpret_cast<const volatile uint32_t*>(err) != 0u) return;
  const int64_t nvec = n >> 3;  // 8 elements per thread-iteration → one 16-byte bf16 store per peer
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    float outv[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t j = i * 2 + h;
      float4 twv[kMaxPeers];  // all peer loads in flight before the first use
#pragma unroll
      for (int w = 0; w < kMaxPeers; ++w)
        if (w < thetas.n) twv[w] = ld_relaxed_sys_f4(reinterpret_cast<const float4*>(thetas.p[w]) + j);
      float4 t0 = reinterpret_cast<const float4*>(theta0)[j];
      float4 mm = reinterpret_cast<const float4*>(mom)[j];
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int w = 0; w < kMaxPeers; ++w) {
        if (w < thetas.n) {
          const float4 tw = twv[w];
          g.x += t0.x - tw.x, g.y += t0.y - tw.y, g.z += t0.z - tw.z, g.w += t0.w - tw.w;
        }
      }
      float* tp = &t0.x;
      float* mp = &mm.x;
      const float* gp = &g.x;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float gk = gp[k] * a.inv_workers;
        const float mk = a.momentum * mp[k] + gk;
        mp[k] = mk;
        const float upd = a.nesterov ? gk + a.momentum * mk : mk;
        tp[k] = tp[k] - a.lr * upd;
        outv[h * 4 + k] = tp[k];
      }
      reinterpret_cast<float4*>(theta0)[j] = t0;
      reinterpret_cast<float4*>(mom)[j] = mm;
      reinterpret_cast<float4*>(theta_new)[j] = t0;
    }
    const int64_t d0 = table_dst(tab, i * 8);
    const bf16x8 pk = pack8(outv);
#pragma unroll
    for (int qd = 0; qd < kMaxPeers; ++qd)
      if (qd < dst.n) stg_v4(reinterpret_cast<bf16x8*>(reinterpret_cast<__nv_bfloat16*>(dst.p[qd]) + d0), pk);
  }
}
PB_EXPORT int pb_outer_nesterov_f32(const PeerPtrs* thetas, float* theta0, float* mom, float* theta_new, int64_t n, const OuterArgs* a,
                                    const PeerPtrs* dst, const int64_t* shard_start, const int64_t* dst_start, int nb,
                                    const uint32_t* err, cudaStream_t stream) {
  if (n % 8 != 0 || nb < 1) return -1;
  BucketTable tab{shard_start, dst_start, nb};
  outer_nesterov_f32_kernel<<<132 * 4, 256, 0, stream>>>(*thetas, theta0, mom, theta_new, n, *a, *dst, tab, err);
  PB_CHECK_LAUNCH();
  return 0;
}

// fp32 master → bf16 parameter buffers of every FSDP peer (used after checkpoint load / outer f32 path).
__global__ void __launch_bounds__(512) cast_push_kernel(const float* __restrict__ src, int64_t n, PeerPtrs dst,
                                                        int64_t dst_off) {
  const int64_t nvec = n >> 3;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(src)[2 * i], b = reinterpret_cast<const float4*>(src)[2 * i + 1];
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    const bf16x8 pk = pack8(f);
#pragma unroll
    for (int q = 0; q < kMaxPeers; ++q)
      if (q < dst.n) stg_v4(reinterpret_cast<bf16x8*>(reinterpret_cast<__nv_bfloat16*>(dst.p[q]) + dst_off) + i, pk);
  }
}
PB_EXPORT int pb_cast_push(const float* src, int64_t n, const PeerPtrs* dst, int64_t dst_off, cudaStream_t stream) {
  if (n % 8 != 0 || dst_off % 8 != 0) return -1;
  cast_push_kernel<<<132 * 2, 512, 0, stream>>>(src, n, *dst, dst_off);
  PB_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// NVLS in-place all-reduce over the multicast mapping (parallel/multicast.py: MulticastHeap.all_reduce_).
// ------------------------------------------------------------------------------------------------
// All-ranks barrier for ONE block index: every rank's block `b` adds 1 to flag[b] on every GPU with a single multimem.red,
// then waits on its own copy until `world` arrivals of this phase are in. Counters only grow: phase k of launch `epoch`
// (k = 0 arrive, 1 depart) completes at world·(2·(epoch-1) + k + 1), so no reset and no ABA across launches.
// Returns false in every thread of the block when the wait failed (timeout or host abort, recorded in the error word).
__device__ __forceinline__ bool mc_barrier(uint32_t* mc_flags, const uint32_t* local_flags, uint32_t target, uint32_t* err) {
  __shared__ int s_ok;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    mc_red_release_add_u32(mc_flags + blockIdx.x, 1u);
    s_ok = spin_wait_ge(local_flags + blockIdx.x, target, err);
  }
  __syncthreads();
  return s_ok;
}

// n16 = number of 16-byte units; each rank owns a contiguous 1/world of them: it reduces that slice through the switch and
// multicasts it back, so the all-reduce is two-shot in one kernel.
template <bool BF16>
__global__ void __launch_bounds__(512) mc_all_reduce_kernel(void* mc, int64_t n16, uint32_t* mc_flags, const uint32_t* local_flags,
                                                             int rank, int world, uint32_t epoch, uint32_t* err) {
  const uint32_t base = (uint32_t)world * 2u * (epoch - 1u);
  if (!mc_barrier(mc_flags, local_flags, base + (uint32_t)world, err)) return;  // a rank's input never arrived: reduce nothing
  const int64_t per = (n16 + world - 1) / world;
  const int64_t lo = per * rank, hi = lo + per < n16 ? lo + per : n16;
  uint4* p = reinterpret_cast<uint4*>(mc);
  for (int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (int64_t)gridDim.x * blockDim.x) {
    if constexpr (BF16) {
      const uint4 v = mc_ld_reduce_bf16x8(p + i);
      mc_st_bf16x8(p + i, v);
    } else {
      const float4 v = mc_ld_reduce_f32x4(reinterpret_cast<const float*>(p + i));
      mc_st_f32x4(reinterpret_cast<float*>(p + i), v);
    }
  }
  mc_barrier(mc_flags, local_flags, base + 2u * (uint32_t)world, err);  // every slice has been written everywhere
}

// Number of flag words an all-reduce needs (one per block) — the grid is fixed so that every rank launches the same one
// and all blocks are co-resident (a spinning block must never wait for a partner that is queued behind it).
PB_EXPORT int pb_mc_all_reduce_grid() { return 132; }

// dtype: 0 = f32, 1 = bf16. `mc_data` and `mc_flags` are addresses in the MULTICAST mapping, `local_flags` the same words
// in this rank's unicast mapping. nbytes must be a multiple of 16. `epoch` starts at 1 and grows by 1 per call on every rank.
PB_EXPORT int pb_mc_all_reduce(void* mc_data, int64_t nbytes, int dtype, uint32_t* mc_flags, const uint32_t* local_flags, int rank,
                               int world, uint32_t epoch, uint32_t* err, cudaStream_t stream) {
  if (nbytes % 16 != 0 || epoch == 0 || world < 1) return -1;
  const int grid = pb_mc_all_reduce_grid();
  if (dtype == 1)
    mc_all_reduce_kernel<true><<<grid, 512, 0, stream>>>(mc_data, nbytes / 16, mc_flags, local_flags, rank, world, epoch, err);
  else if (dtype == 0)
    mc_all_reduce_kernel<false><<<grid, 512, 0, stream>>>(mc_data, nbytes / 16, mc_flags, local_flags, rank, world, epoch, err);
  else
    return -1;
  PB_CHECK_LAUNCH();
  return 0;
}
