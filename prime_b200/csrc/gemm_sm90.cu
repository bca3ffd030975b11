// bf16 GEMM for sm_90a: TMA → 128B-swizzled shared memory → wgmma (accumulators in registers) → epilogue staged through shared
// memory and written by TMA stores (GEMM ⊕ reduce-scatter: fp32 atomics from registers into the owner rank's buffer).
// Persistent, warp-specialised, one CTA per SM.
//
//   C[M,N] (bf16 | fp32, optional +=)  =  A ⋅ Bᵀ   with fp32 accumulation
//     A: "K-major"  stored [M,K] (K contiguous)   or "MN-major" stored [K,M] (M contiguous)
//     B: "K-major"  stored [N,K] (K contiguous)   or "MN-major" stored [K,N] (N contiguous)
//
// The three linear-layer GEMMs map onto this without any transposes in memory:
//     y  = x  Wᵀ      : A=x  (K-major)   B=W  (K-major)
//     dx = dy W       : A=dy (K-major)   B=W  (MN-major)
//     dW = dyᵀ x      : A=dy (MN-major)  B=x  (MN-major)     (fp32 accumulate into main_grad)
//
// Tile 128 x BN x 64. BN = 128: 6-stage TMA ring (32 KB / stage; 5 stages when the weight-gather copier takes 32 KB).
// BN = 256 (local GEMMs only, IO = 0): 4 stages of 48 KB; the producer warpgroup drops to 40 registers and the consumer
// warpgroups rise to 232 (setmaxnreg) to hold 128 fp32 accumulators per thread. tile_policy() picks BN from the shape.
// Warp roles: warpgroup 0 = w0 TMA producer (1 lane), w3 gather copier (IO = 1 / 3); warpgroups 1 and 2 = consumers, each
// issuing m64nBNk16 wgmma for 64 rows of the tile and running the epilogue of those rows, while the producer already fills
// the ring for the next tile (see kOutSlots).
#include <cuda.h>

#include "common.cuh"
#include "tc_common.cuh"
#include "tmap.h"

// Fused epilogue of pb_gemm_bf16 / pb_gemm_wgather; a null descriptor means plain. Mirrored by ops/_lib.py: GemmEpilogue.
struct GemmEpilogue {
  int kind;  // 0 plain, 1 RoPE, 2 SwiGLU, 3 SwiGLU backward
  // RoPE (the fused QKV projection): output columns [0, rope_cols) are heads of width rope_D (64 | 128); output row r is token r
  // of a [B, rope_S] batch; cos / sin are fp32 [>= rope_S, rope_D/2]
  const float* rope_cos;
  const float* rope_sin;
  int rope_S, rope_cols, rope_D;
  // SwiGLU: h [M, FF] (written); SwiGLU backward: the saved gate_up [M, 2·FF] (read)
  void* aux;
  int ld_aux;
};

namespace {

constexpr int BM = 128, BN = 128, BK = 64;  // BN: the narrow tile, the only one of the collective variants
constexpr int kWideBN = 256;
constexpr int kThreads = 384;
constexpr int kConsumerWarps = 8;
constexpr uint32_t kABytes = BM * BK * 2;  // 16 KB
constexpr int kGroupM = 16;  // raster: super-rows of 16 M-tiles keep the A slab L2-resident
constexpr int kAgIdleRounds = 2;  // IO = 1: scheduling rounds a CTA sits out after a gather tile (it costs several ordinary tiles)

constexpr uint32_t kCopyChunkBytes = 128 * BK * 2;  // IO = 3 weight-gather copier: one {64 col, 128 row} box = 16 KB
constexpr int kCopyBufs = 2;
constexpr int kGatherSub = 4;  // IO = 3: readiness flags per rank block (a block is released to the MMA tiles in quarters)

// Epilogue staging (every IO mode but the reduce-scatter): each consumer warpgroup owns kOutSlots slots of 64 rows x 64 B, the
// box of a 64B-swizzled output tensor map (32 bf16 or 16 fp32 columns). The epilogue writes a step of slots, one elected thread
// TMA-stores them, and the warpgroup goes on without waiting for the global writes.
constexpr int kOutSlots = 4;
constexpr uint32_t kSlotBytes = 64 * 64;

template <int IO, int TBN>
struct Geo {
  static constexpr int kStages = TBN == kWideBN ? 4 : IO == 3 ? 5 : 6;
  static constexpr uint32_t kBBytes = TBN * BK * 2;  // 16 | 32 KB
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  static constexpr uint32_t kCopyBytes = IO == 3 ? kCopyBufs * kCopyChunkBytes : 0;
  static constexpr uint32_t kOutBytes = IO != 2 ? 2 * kOutSlots * kSlotBytes : 0;
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + kCopyBytes + kOutBytes + 1024 /*align slack*/ + 512 /*barriers*/;
};
static_assert(Geo<0, kWideBN>::kSmemBytes <= 227 * 1024, "wide tile ring + epilogue staging exceed the shared memory of an SM");
static_assert(Geo<0, BN>::kSmemBytes <= 227 * 1024, "narrow tile ring + epilogue staging exceed the shared memory of an SM");
static_assert(Geo<1, BN>::kSmemBytes <= 227 * 1024, "all-gather ring + epilogue staging exceed the shared memory of an SM");
static_assert(Geo<2, BN>::kSmemBytes <= 227 * 1024, "reduce-scatter ring exceeds the shared memory of an SM");
static_assert(Geo<3, BN>::kSmemBytes <= 227 * 1024, "weight-gather ring + copier + epilogue staging exceed the shared memory of an SM");

using namespace tc;

__device__ __forceinline__ void tile_coords(int tile, int tiles_m, int tiles_n, int& tm, int& tn) {
  const int per_group = kGroupM * tiles_n;
  const int g = tile / per_group;
  const int first_m = g * kGroupM;
  const int gsz = min(kGroupM, tiles_m - first_m);
  const int r = tile - g * per_group;
  tm = first_m + r % gsz;
  tn = r / gsz;
}

struct GemmParams {
  int M, N, K;
  int ldc;
  int a_mn, b_mn;
  int c_fp32, accumulate;
  int split_k;  // >1 only with c_fp32 && accumulate: every K slice atomically adds its partial tile (weight-gradient GEMMs)
  void* C;  // read by the bf16 += only; the staged epilogue writes through EpiMaps
  // RoPE (EPI = 1, the QKV projection): output columns [0, rope_cols) are heads of width rope_D whose interleaved pairs are rotated
  // by the position (row % rope_S) while the tile is still in registers. The kernel reads the RoPE fields only.
  GemmEpilogue epi;
  // SwiGLU (EPI = 2, gate/up projection): B = W13 stored [2·FF, K] as [gate rows | up rows]; a tile covers 64 features: the
  // producer stages the 64 GATE rows and the matching 64 UP rows, so every thread holds gate and up of the same (row, feature) in
  // accumulator columns j and j + 64. The epilogue stores gate and up (bf16, for the backward) into C = gate_up [M, 2·FF] and
  // h = silu(gate)·up into h [M, FF].
  // SwiGLU backward (EPI = 3, the down-projection's input-gradient GEMM dh = dy·W2, N = FF): the epilogue reads the saved bf16
  // gate/up of the same (row, feature) from gate_up [M, 2·FF] and stores d_gate = dh·up·silu'(gate) and d_up = dh·silu(gate) into
  // C = d_gate_up [M, 2·FF] — dh never exists in memory.
  int swiglu_ff;
};

// The staged epilogue's 64B-swizzled tensor maps (see kOutSlots), for every IO mode but the reduce-scatter.
struct EpiMaps {
  CUtensorMap c;   // C [M, N] (SwiGLU backward: d_gate_up [M, 2·N]), bf16 or fp32
  CUtensorMap h;   // EPI = 2: h [M, FF]
  CUtensorMap gu;  // EPI = 3: the saved gate_up [M, 2·FF] (read)
};

// Fused collective GEMMs over the NVLink symmetric heap (IO template parameter of the kernel):
//   IO = 1  all-gather ⊕ GEMM : row block r of A lives on rank r. Peer memory is NOT cached in the local L2, so a remote A tile
//           must cross NVLink exactly once: the tiles of output column 0 of every remote row block ("gather tiles", scheduled
//           first, owners interleaved) TMA-load their A tiles straight from the owner into the MMA ring, and an otherwise idle
//           warp TMA-stores each consumed ring slot into a local gathered copy of A; a per-row-block flag then releases the
//           remaining column tiles of that block, which read the local copy (L2-resident). Local row blocks are scheduled between
//           the two, so the NVLink transfer hides behind them.
//   IO = 2  GEMM ⊕ reduce-scatter : every rank computes a full partial C; the epilogue atomically adds each fp32 element into the
//           buffer of the rank that owns those rows (peer-mapped address). Row blocks are visited owner-interleaved
//           (rank+1, rank+2, …, self) so the NVLink reduce traffic is spread over the whole kernel.
//   IO = 3  parameter all-gather ⊕ GEMM (ZeRO-3 / reshard_after_forward): the WEIGHT (operand B, stored [rows, cols]) is sharded by
//           rows over the ranks of the FSDP group — rank r owns rows [r·rpr, (r+1)·rpr) in its symmetric-heap shard. Nothing is
//           gathered ahead of the kernel: warp 3 of EVERY CTA is a copier that TMA-loads {64 x 128} boxes of the peers' shards
//           over NVLink into a 16 KB bounce buffer and TMA-stores them into a local full-size copy of the weight, walking the rank
//           blocks in consumption order (own block first); a per-quarter-block counter releases the MMA tiles, whose TMA producer
//           waits on the counters of exactly the B rows it is about to load and reads them from the local copy (L2-resident).
//           K-major B (forward): the output-column order is rotated to start at the own block; MN-major B (input gradient, the
//           contraction runs over the sharded rows): the K loop is rotated instead. The shards are read-only during
//           forward/backward, so no inter-rank barrier is needed around the kernel.
struct PeerMaps {
  CUtensorMap m[8];   // IO = 1: the ranks' blocks of A; IO = 3: the ranks' shards of the weight
  float* c[8];        // IO = 2: the ranks' fp32 output buffers as mapped in this process
  int n;              // ranks
  int rows_per_rank;  // IO 1/2: multiple of the tile height; IO 3: rows of B owned by each rank
  int rank;
  uint32_t* flags;    // IO = 1: one counter per 128-row block of the gathered A (zeroed by the host before the launch)
                      // IO = 3: n * kGatherSub counters (chunks landed per quarter block), zeroed before the launch
  // IO = 3
  int order[8];       // rank blocks in the order the copiers fetch them (= the order the tiles consume them)
  int cpr;            // 128-row chunk rows per rank block = ceil(rows_per_rank / 128)
  int col_chunks;     // cols / 64
  int spc;            // chunk rows per readiness counter = ceil(cpr / kGatherSub)
  int start;          // first output-column tile (K-major B) / first k-block (MN-major B) of the rotated order
  int gate;           // 1: B is gathered by THIS kernel and the tiles wait for it; 0: B is already resident in the local scratch
  // gather-AHEAD list: the weight the NEXT GEMM of the layer sequence consumes (forward: wqkv → wo → w13 → w2 → next layer;
  // backward: the reverse dgrad order). After (or instead of) its own weight the copier pulls this one into ITS scratch region, so
  // the next kernel finds its operand resident and runs un-gated: in steady state every gather hides under the previous GEMM and
  // only the first kernel of a pass waits for NVLink.
  CUtensorMap nm[8];
  int nn;             // ranks holding the next weight (0 = nothing to prefetch)
  int ncpr, ncol_chunks;
  int norder[8];
};
// the kernel's parameters: four operand maps, GemmParams (padded to the maps' 64-byte alignment), EpiMaps and PeerMaps
static_assert(4 * sizeof(CUtensorMap) + (sizeof(GemmParams) + 63) / 64 * 64 + sizeof(EpiMaps) + sizeof(PeerMaps) <= 4096,
              "gemm_bf16_kernel's parameters exceed 4 KB");

// IO = 1 tile schedule: [gather tiles][local tiles][dependent tiles]; kind 1 = gather (tn = 0 of a remote block), 0 = local rows,
// 2 = dependent (waits for the block's flag, reads the local gathered copy). Lower indices never wait on higher ones.
__device__ __forceinline__ void ag_tile(int idx, const PeerMaps& pm, int tiles_n, int tpr, int& tm, int& tn, int& kind) {
  const int n = pm.n, G = (n - 1) * tpr, L = tpr * tiles_n;
  if (idx < G) {
    tm = ((pm.rank + 1 + idx % (n - 1)) % n) * tpr + idx / (n - 1);
    tn = 0;
    kind = 1;
  } else if (idx < G + L) {
    const int j = idx - G;
    tm = pm.rank * tpr + j % tpr;
    tn = j / tpr;
    kind = 0;
  } else {
    const int j = idx - G - L, g = j % G;
    tm = ((pm.rank + 1 + g % (n - 1)) % n) * tpr + g / (n - 1);
    tn = 1 + j / G;
    kind = 2;
  }
}
// IO = 1 static schedule with load balancing: iteration `it` of CTA `sched_id` → tile index, -1 = idle slot, -2 = done.
// Round 0 hands gather tile p to CTA p < G; those CTAs then sit out kAgIdleRounds rounds while the others keep taking tiles.
__device__ __forceinline__ int ag_next(int it, int sched_id, int sched_n, int G, int num_tiles) {
  constexpr int idle = kAgIdleRounds;
  if (G == 0 || G > sched_n) {
    const int t = sched_id + it * sched_n;
    return t < num_tiles ? t : -2;
  }
  const int R = num_tiles - G;  // non-gather tiles, numbered in order behind the gather tiles
  int r;
  if (it == 0) {
    if (sched_id < G) return sched_id;
    r = sched_id - G;
  } else if (it <= idle) {
    if (sched_id < G) return -1;
    r = (sched_n - G) * it + (sched_id - G);
  } else {
    r = (sched_n - G) * (idle + 1) + (it - idle - 1) * sched_n + sched_id;
  }
  return r < R ? G + r : -2;
}
// IO = 2 row-block order: raster index t → owner-interleaved tile row
__device__ __forceinline__ int rs_tile_row(int t, const PeerMaps& pm, int tpr) { return ((pm.rank + 1 + t % pm.n) % pm.n) * tpr + t / pm.n; }

// EPI: 0 = plain, 1 = RoPE on the leading output columns, 2 = SwiGLU, 3 = SwiGLU backward. Separate instantiations on purpose: the
// fused epilogues need more registers, and a plain GEMM compiled with that footprint leaves less of the register file to the
// gradient-reduction / optimizer kernels of the comm stream that co-reside with it during the backward pass.
// TBN: tile width, BN or kWideBN (IO = 0 only). tmap_g: IO = 3 the local full-weight copy; IO = 0 wide SwiGLU the up rows of W13
// (tmap_b then covers the FF gate rows only, so the TMA unit zero-fills a last tile that is half past FF).
template <int A_MN, int B_MN, int EPI, int IO, int TBN>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                     const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_g2, const GemmParams p,
                     const __grid_constant__ EpiMaps em, const __grid_constant__ PeerMaps pm) {
  static_assert(TBN == BN || (TBN == kWideBN && IO == 0), "the wide tile exists for local GEMMs only");
  static_assert(IO != 1 || EPI == 0, "all-gather ⊕ GEMM has no fused epilogue (its ag_next order would break the gate_up cursor)");
  constexpr bool wide = TBN == kWideBN;
  using G = Geo<IO, TBN>;
  constexpr int kStages = G::kStages;
  constexpr uint32_t kStageBytes = G::kStageBytes;
  const int sched_id = (int)blockIdx.x;
  const int sched_n = (int)gridDim.x;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* copy_buf = smem + kStages * kStageBytes;  // IO = 3: kCopyBufs x 16 KB bounce buffers of the weight-gather copier
  uint8_t* out_buf = copy_buf + G::kCopyBytes;  // IO != 2: 2 x kOutSlots epilogue staging slots
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(out_buf + G::kOutBytes);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* copied_bar = empty_bar + kStages;  // IO = 1: the gather copier has finished reading a consumed ring slot
  uint64_t* cp_bar = copied_bar + kStages;     // IO = 3: a peer box has landed in bounce buffer i
  uint64_t* aux_bar = cp_bar + kCopyBufs;      // SwiGLU backward: gate / up boxes landed in slot pair 2·wg + half

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr bool swiglu = EPI == 2;
  // SwiGLU: a tile covers TBN / 2 features (the gate and the up rows of each)
  const int tiles_m = (p.M + BM - 1) / BM;
  const int tiles_n = swiglu ? (wide ? (p.swiglu_ff + TBN / 2 - 1) / (TBN / 2) : p.swiglu_ff / 64) : (p.N + TBN - 1) / TBN;
  const int num_kb = (p.K + BK - 1) / BK;
  // split-K: work item w = tile * split_k + slice; slice s covers k-blocks [s*kb_per, min(num_kb, (s+1)*kb_per))
  const int split_k = p.split_k;
  const int kb_per = (num_kb + split_k - 1) / split_k;
  const int num_tiles = tiles_m * tiles_n * split_k;  // = number of work items
  const int ag_G = (IO == 1 && pm.n > 1) ? (pm.n - 1) * (pm.rows_per_rank / BM) : 0;  // gather tiles (lowest indices)
  // every role walks the same tile sequence: round-robin over the CTAs; all-gather mode inserts idle slots (ag_next)
  auto next_tile = [&](int& it) -> int {
    if (IO == 1 && pm.n > 1) {
      for (;;) {
        const int t = ag_next(it++, sched_id, sched_n, ag_G, num_tiles);
        if (t != -1) return t;
      }
    }
    const int t = sched_id + (it++) * sched_n;
    return t < num_tiles ? t : -2;
  };
  // IO = 3 rotations (see PeerMaps): K-major B → output columns start at the own rank block; MN-major B → the K loop does
  const int tn_rot = (IO == 3 && B_MN == 0 && pm.gate) ? pm.start : 0;
  const int kb_rot = (IO == 3 && B_MN == 1 && pm.gate) ? pm.start : 0;
  const int tpr = IO != 0 ? pm.rows_per_rank / BM : 0;  // tile rows per rank
  auto coords = [&](int tile, int& tm, int& tn, int& kind) {
    kind = 0;
    if (IO == 1 && pm.n > 1) {
      ag_tile(tile, pm, tiles_n, tpr, tm, tn, kind);
    } else {
      tile_coords(tile / split_k, tiles_m, tiles_n, tm, tn);
      if (IO == 2) tm = rs_tile_row(tm, pm, tpr);
      if (IO == 3 && tn_rot) tn = (tn + tn_rot) % tiles_n;
    }
  };

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    if (IO == 3) {
      prefetch_tmap(&tmap_g);
      prefetch_tmap(&tmap_g2);
    }
    if (IO == 1 || IO == 3)
      for (int i = 0; i < pm.n; ++i) prefetch_tmap(&pm.m[i]);
    if (IO != 2) {  // the staged epilogue's maps
      prefetch_tmap(&em.c);
      if (EPI == 2) prefetch_tmap(&em.h);
      if (EPI == 3) prefetch_tmap(&em.gu);
    }
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumerWarps);  // one arrive per consumer warp
      mbar_init(&copied_bar[i], 1);
    }
    for (int i = 0; i < kCopyBufs; ++i) mbar_init(&cp_bar[i], 1);
    if (EPI == 3)
      for (int i = 0; i < 4; ++i) mbar_init(&aux_bar[i], 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0 || (wide && warp < 4)) {
    // ------------------------------------------------------------------ TMA producer
    // wide tile: the whole warpgroup hands registers to the consumers; lane 0 of warp 0 is the producer
    if constexpr (wide) setmaxnreg_dec<40>();
    if (lane == 0 && (!wide || warp == 0)) {
      int stage = 0;
      uint32_t phase = 0;
      // gather tiles have the lowest indices: this CTA's are tiles sched_id, sched_id + sched_n, … below G
      const int gather_fills = ag_G > sched_id ? ((ag_G - sched_id + sched_n - 1) / sched_n) * num_kb : 0;
      int fill = 0;
      // IO = 3: wait until the copiers have landed B rows [r0, r1] in the local full copy. One readiness counter per quarter of a
      // rank block; a counter that was seen complete stays complete for the rest of the kernel (bit in `ready`).
      uint32_t ready = 0;
      auto gate_rows = [&](int r0, int r1) {
        if (IO != 3 || !pm.gate) return;
        const int rpr = pm.rows_per_rank;
        for (int x = r0; x <= r1;) {
          const int b = x / rpr, cr = (x - b * rpr) >> 7;
          const int q = min(cr / pm.spc, kGatherSub - 1);
          const int id = b * kGatherSub + q;
          const int cr_end = q == kGatherSub - 1 ? pm.cpr : min(pm.cpr, (q + 1) * pm.spc);  // chunk rows [q*spc, cr_end)
          if (!((ready >> id) & 1u)) {
            const uint32_t expect = (uint32_t)((cr_end - q * pm.spc) * pm.col_chunks);
            SpinGuard guard;
            while (pb::ld_acquire_gpu_u32(pm.flags + id) < expect) guard.tick();
            fence_proxy_async_all();  // generic-proxy acquire → the TMA (async-proxy) reads of those rows
            ready |= 1u << id;
          }
          x = b * rpr + min(rpr, cr_end * 128);  // first row of the next quarter (or of the next rank block)
        }
      };
      const int rows_b = pm.rows_per_rank * pm.n;
      for (int it = 0, tile; (tile = next_tile(it)) >= 0;) {
        int tm, tn, kind;
        coords(tile, tm, tn, kind);
        const int kb0 = (tile % split_k) * kb_per, kb1 = min(num_kb, kb0 + kb_per);
        if (kb0 >= kb1) continue;  // empty K slice (split does not divide K): every role skips it identically
        const int m0 = tm * BM;
        // SwiGLU: TBN / 2 gate rows and the matching up rows; otherwise TBN consecutive B rows
        const int n0 = swiglu ? tn * (TBN / 2) : tn * TBN;
        if (IO == 3 && B_MN == 0) {  // my B rows have landed locally
          if (swiglu) {
            gate_rows(n0, min(n0 + 64, rows_b) - 1);
            gate_rows(p.swiglu_ff + n0, min(p.swiglu_ff + n0 + 64, rows_b) - 1);
          } else {
            gate_rows(n0, min(n0 + BN, rows_b) - 1);
          }
        }
        if (IO == 1 && kind == 2) {  // the block's gather tile has stored these rows locally
          SpinGuard guard;
          while (pb::ld_acquire_gpu_u32(pm.flags + tm) < 1u) guard.tick();
          fence_proxy_async_all();  // generic-proxy acquire → the TMA (async-proxy) reads below
        }
        for (int kbi = kb0; kbi < kb1; ++kbi) {
          const int kb = kb_rot ? (kbi + kb_rot) % num_kb : kbi;
          if (IO == 3 && B_MN == 1) gate_rows(kb * BK, min(kb * BK + BK, rows_b) - 1);
          mbar_wait(&empty_bar[stage], phase ^ 1);
          // the slot's previous fill was a gather fill (they are the first fills of every CTA): the copier must have drained it
          if (IO == 1 && fill >= kStages && fill - kStages < gather_fills) mbar_wait(&copied_bar[stage], phase ^ 1);
          ++fill;
          uint8_t* sa = smem + stage * kStageBytes;
          uint8_t* sb = sa + kABytes;
          mbar_expect_tx(&full_bar[stage], kStageBytes);
          auto load = [&](const CUtensorMap* m, void* dst, int c0, int c1) { tma_load_2d(m, &full_bar[stage], dst, c0, c1); };
          if (IO == 1) {
            // gather / local tiles read the owner's block (NVLink for remote owners); dependent tiles read the local gathered copy
            const int owner = m0 / pm.rows_per_rank;
            if (kind == 2) load(&tmap_a, sa, kb * BK, m0);
            else load(&pm.m[owner], sa, kb * BK, m0 - owner * pm.rows_per_rank);
          } else if (A_MN == 0) {
            load(&tmap_a, sa, kb * BK, m0);  // box {64 k, 128 m}
          } else {
#pragma unroll
            for (int j = 0; j < BM / 64; ++j)  // box {64 m, 64 k} → 8 KB each
              load(&tmap_a, sa + j * (BK * 128), m0 + j * 64, kb * BK);
          }
          if (swiglu && wide) {  // boxes {64 k, 128 n}: gate rows, then the matching up rows, each from its own FF-row map
            load(&tmap_b, sb, kb * BK, n0);
            load(&tmap_g, sb + 128 * 128, kb * BK, n0);
          } else if (swiglu) {  // boxes {64 k, 64 n}: gate rows, then the matching up rows
            load(&tmap_b, sb, kb * BK, n0);
            load(&tmap_b, sb + 64 * 128, kb * BK, p.swiglu_ff + n0);
          } else if (B_MN == 0) {
            load(&tmap_b, sb, kb * BK, n0);  // box {64 k, TBN n}
          } else {
#pragma unroll
            for (int j = 0; j < TBN / 64; ++j)
              load(&tmap_b, sb + j * (BK * 128), n0 + j * 64, kb * BK);
          }
          if (++stage == kStages) stage = 0, phase ^= 1;
        }
      }
    }
  } else if (IO == 1 && warp == 3) {
    // ------------------------------------------------------------------ gather copier (all-gather ⊕ GEMM only)
    // follows the ring in consumption order: once the consumers have retired a slot (empty barrier), a gather tile's A slab is
    // TMA-stored into the local gathered copy before the producer may refill the slot; after the tile, the block's flag is bumped
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int it = 0, tile; (tile = next_tile(it)) >= 0;) {
        int tm = 0, tn = 0, kind = 0;
        if (pm.n > 1) ag_tile(tile, pm, tiles_n, tpr, tm, tn, kind);
        if (kind != 1) break;  // gather tiles come first; nothing to copy afterwards (the producer stops waiting for us too)
        const int m0 = tm * BM;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase);
          tma_store_2d(&tmap_a, smem + stage * kStageBytes, kb * BK, m0);
          bulk_commit();
          bulk_wait_read<0>();
          mbar_arrive(&copied_bar[stage]);
          if (++stage == kStages) stage = 0, phase ^= 1;
        }
        bulk_wait_all();          // the rows are in local memory …
        fence_proxy_async_all();  // … async-proxy writes ordered before the generic-proxy release below
        pb::red_add_release_gpu_u32(pm.flags + tm, 1u);
      }
    }
  } else if (IO == 3 && warp == 3) {
    // ------------------------------------------------------------------ weight-gather copier (parameter all-gather ⊕ GEMM)
    // Every CTA of the grid takes the {64 col x 128 row} boxes g = blockIdx.x, blockIdx.x + gridDim.x, … of the whole weight in
    // consumption order: peer shard --TMA load (NVLink)--> bounce buffer --TMA store--> local full copy, then bumps the
    // readiness counter of the box's quarter block once the store has fully completed. Two boxes are in flight per CTA.
    if (lane == 0) {
      uint32_t ph = 0;  // bit i: the phase of bounce buffer i (a bit mask, not an array: no stack frame)
      // one list = one weight: (peer maps, local store map, rank order, geometry); `flags` != nullptr → publish per-quarter counters
      auto gather_list = [&](const CUtensorMap* maps, const CUtensorMap* store_map, const int* order, int n, int cpr, int col_chunks,
                             int spc, uint32_t* flags) {
        const int cpb = cpr * col_chunks;  // boxes per rank block
        const int total = cpb * n;
        const int mine = total > (int)blockIdx.x ? (total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
        auto box = [&](int i, int& owner, int& cr, int& cc) {
          const int g = (int)blockIdx.x + i * (int)gridDim.x;
          const int j = g / cpb, c = g - j * cpb;
          owner = order[j];
          cr = c / col_chunks;
          cc = c - cr * col_chunks;
        };
        auto fetch = [&](int i) {  // rows past the end of the owner's shard are zero-filled by the TMA unit
          int owner, cr, cc;
          box(i, owner, cr, cc);
          const int buf = i % kCopyBufs;
          mbar_expect_tx(&cp_bar[buf], kCopyChunkBytes);
          tma_load_2d(&maps[owner], &cp_bar[buf], copy_buf + buf * kCopyChunkBytes, cc * BK, cr * 128);
        };
        for (int i = 0; i < kCopyBufs && i < mine; ++i) fetch(i);  // both NVLink loads in flight from the start
        int prev_id = -1;
        for (int i = 0; i < mine; ++i) {
          int owner, cr, cc;
          box(i, owner, cr, cc);
          const int buf = i % kCopyBufs;
          mbar_wait(&cp_bar[buf], (ph >> buf) & 1u);
          ph ^= 1u << buf;
          // … and clipped by the store: dimension 1 of the 3-D map is the rows of ONE rank block
          tma_store_3d(store_map, copy_buf + buf * kCopyChunkBytes, cc * BK, cr * 128, owner);
          bulk_commit();
          if (flags != nullptr && prev_id >= 0) {  // the previous box's WRITES are complete (not only its smem reads): publish it
            asm volatile("cp.async.bulk.wait_group 1;" ::: "memory");
            fence_proxy_async_all();
            pb::red_add_release_gpu_u32(flags + prev_id, 1u);
          }
          prev_id = owner * kGatherSub + min(cr / spc, kGatherSub - 1);
          if (i + kCopyBufs < mine) {
            bulk_wait_read<0>();  // this buffer has been read out by the store above
            fetch(i + kCopyBufs);
          }
        }
        bulk_wait_all();  // every box of this list is in local memory (the NEXT kernel relies on that for a gather-ahead list)
        if (flags != nullptr && prev_id >= 0) {
          fence_proxy_async_all();
          pb::red_add_release_gpu_u32(flags + prev_id, 1u);
        }
      };
      if (pm.gate) gather_list(pm.m, &tmap_g, pm.order, pm.n, pm.cpr, pm.col_chunks, pm.spc, pm.flags);
      if (pm.nn > 0) gather_list(pm.nm, &tmap_g2, pm.norder, pm.nn, pm.ncpr, pm.ncol_chunks, 1, nullptr);
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumers: wgmma main loop + epilogue
    if constexpr (wide) setmaxnreg_inc<232>();
    const int wg = (warp - 4) >> 2;  // rows [wg*64, wg*64 + 64) of the tile
    const int wi = warp & 3;         // warp inside the warpgroup: accumulator rows wi*16 + lane/4 (+8)
    int stage = 0;
    uint32_t phase = 0;
    float acc[TBN / 2];
    // staged epilogue: this warpgroup's slots, its leader (the one thread that issues TMA), the swizzle key of this thread's rows
    // (rows r and r + 8 share it), the slot offset of row r, and the count of double-buffered steps so far
    uint8_t* slots = out_buf + wg * (kOutSlots * kSlotBytes);
    const bool leader = IO != 2 && (threadIdx.x & 127) == 0;
    const uint32_t skey = (lane >> 3) & 3;
    const uint32_t roff = (wi * 16 + (lane >> 2)) * 64;
    uint32_t ostep = 0;
    // SwiGLU backward: the leader TMA-loads the gate / up boxes of the step two ahead of the one the warpgroup is working on, in
    // the step order of the tile sequence, so the first two steps of a tile land during its main loop. Cursor: tile, step.
    // The cursor steps through the tiles in plain round-robin order, which is next_tile's order for IO = 0 and IO = 3 (whose tn
    // rotation happens inside coords()); IO = 1's ag_next order would break it, and IO = 1 has no fused epilogue.
    int l_it = 0, l_tile = sched_id, l_st = 0;
    uint32_t l_n = 0;
    auto aux_issue = [&] {  // leader: load the cursor's step into slot pair l_n % 2, then advance the cursor
      int tm, tn, kind;
      coords(l_tile, tm, tn, kind);
      const int f0 = tn * TBN + 32 * l_st;
      uint64_t* bar = &aux_bar[2 * wg + (l_n & 1)];
      uint8_t* dst = slots + (l_n & 1) * (2 * kSlotBytes);
      mbar_expect_tx(bar, 2 * kSlotBytes);
      tma_load_2d(&em.gu, bar, dst, f0, tm * BM + wg * 64);
      tma_load_2d(&em.gu, bar, dst + kSlotBytes, p.swiglu_ff + f0, tm * BM + wg * 64);
      ++l_n;
      if (++l_st == TBN / 32 || f0 + 32 >= p.swiglu_ff) l_st = 0, l_tile = sched_id + (++l_it) * sched_n;
    };
    if constexpr (EPI == 3) {
      if (leader)
        for (int i = 0; i < 2 && l_tile < num_tiles; ++i) aux_issue();
    }
    for (int it = 0, tile; (tile = next_tile(it)) >= 0;) {
      int tm, tn, kind;
      coords(tile, tm, tn, kind);
      const int kb0 = (tile % split_k) * kb_per, kb1 = min(num_kb, kb0 + kb_per);
      if (kb0 >= kb1) continue;  // empty K slice
#pragma unroll
      for (int i = 0; i < TBN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * kStageBytes) + wg * (64 * 128);
        const uint32_t sb = smem_u32(smem + stage * kStageBytes) + kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // K-major: +32 B per k16 step inside the 128 B swizzle row.  MN-major: +16 k-rows * 128 B.
          const uint64_t adesc = A_MN == 0 ? make_smem_desc(sa + k * 32, 16, 1024) : make_smem_desc(sa + k * 2048, BK * 128, 1024);
          const uint64_t bdesc = B_MN == 0 ? make_smem_desc(sb + k * 32, 16, 1024) : make_smem_desc(sb + k * 2048, BK * 128, 1024);
          if constexpr (wide) wgmma_m64n256k16<A_MN, B_MN>(acc, adesc, bdesc);
          else wgmma_m64n128k16<A_MN, B_MN>(acc, adesc, bdesc);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's wgmmas have retired: its ring slot may be refilled
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) stage = 0, phase ^= 1;
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      // ---- epilogue: accumulator element acc[4j + i] is row r0 (+8 for i >= 2), column 8j + 2·(lane % 4) (+1 for odd i)
      const int r0 = tm * BM + wg * 64 + wi * 16 + (lane >> 2);
      const int cq = 2 * (lane & 3);
      if constexpr (IO != 2) {
        // Staged: a step writes slots, then the leader TMA-stores them (the unit clips rows >= M and columns past the map).
        const int row0 = tm * BM + wg * 64;
        auto step_begin = [&](bool single) {  // the slots about to be written have been read out by their previous store
          if (leader) {
            if (single) bulk_wait_read<0>();
            else bulk_wait_read<1>();
          }
          named_bar_sync(1 + wg, 128);
        };
        auto step_end = [&] {  // every thread's slot writes → the leader's TMA store
          fence_proxy_async_smem();
          named_bar_sync(1 + wg, 128);
        };
        // byte offset in a slot of this thread's pair in 16-byte chunk jj (0..3), row + 8h; 64B swizzle: chunk ^= (row / 2) % 4
        auto off16 = [&](int jj, int h) { return roff + h * 512 + ((((uint32_t)jj) ^ skey) << 4) + 4 * (lane & 3); };
        // fp32 pair of column group jj (0..1) of a 16-column slot
        auto off32 = [&](int jj, int h) { return roff + h * 512 + (((2u * jj + ((lane & 3) >> 1)) ^ skey) << 4) + 8 * (lane & 1); };
        auto st32 = [&](uint8_t* s, uint32_t v) { *reinterpret_cast<uint32_t*>(s) = v; };
        if constexpr (EPI == 2) {
          const int FF = p.swiglu_ff;
          constexpr int kFeat8 = TBN / 16;  // 8-feature column groups of the gate half; the up half follows
#pragma unroll
          for (int st = 0; st < TBN / 64; ++st) {  // 32 features per step: gate, up and h in slots 0, 1, 2 (single-buffered)
            const int f0 = tn * (TBN / 2) + 32 * st;
            if (f0 >= FF) break;  // FF % 128 = 64: the last wide tile's gate and up halves are half zero-filled
            step_begin(true);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * st + jj;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint32_t gw = pack_bf16(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                const uint32_t uw = pack_bf16(acc[4 * (j + kFeat8) + 2 * h], acc[4 * (j + kFeat8) + 2 * h + 1]);
                // h = silu(gate)·up from the bf16-ROUNDED gate/up — bit-compatible with the stand-alone kernel that reads them back
                const float2 gf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&gw));
                const float2 uf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&uw));
                const float h0 = gf.x / (1.f + __expf(-gf.x)) * uf.x, h1 = gf.y / (1.f + __expf(-gf.y)) * uf.y;
                const uint32_t o = off16(jj, h);
                st32(slots + o, gw);
                st32(slots + kSlotBytes + o, uw);
                st32(slots + 2 * kSlotBytes + o, pack_bf16(h0, h1));
              }
            }
            step_end();
            if (leader) {
              tma_store_2d(&em.c, slots, f0, row0);
              tma_store_2d(&em.c, slots + kSlotBytes, FF + f0, row0);
              tma_store_2d(&em.h, slots + 2 * kSlotBytes, f0, row0);
              bulk_commit();
            }
          }
        } else if constexpr (EPI == 3) {
          const int FF = p.swiglu_ff;
#pragma unroll
          for (int st = 0; st < TBN / 32; ++st) {  // 32 features per step, turned into d_gate / d_up in the slot pair loaded for it
            const int f0 = tn * TBN + 32 * st;
            if (f0 >= FF) break;
            uint8_t* sg = slots + (ostep & 1) * (2 * kSlotBytes);
            mbar_wait(&aux_bar[2 * wg + (ostep & 1)], (ostep >> 1) & 1);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * st + jj;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint32_t o = off16(jj, h);
                const uint32_t gw = *reinterpret_cast<const uint32_t*>(sg + o);
                const uint32_t uw = *reinterpret_cast<const uint32_t*>(sg + kSlotBytes + o);
                const float2 gf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&gw));
                const float2 uf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&uw));
                const float d0 = acc[4 * j + 2 * h], d1 = acc[4 * j + 2 * h + 1];
                // sigmoid through ex2.approx + rcp.approx: IEEE division would make the epilogue longer than the tile's MMAs
                const float s0 = __fdividef(1.f, 1.f + exp2f(-1.4426950408889634f * gf.x));
                const float s1 = __fdividef(1.f, 1.f + exp2f(-1.4426950408889634f * gf.y));
                const float dg0 = d0 * uf.x * s0 * (1.f + gf.x * (1.f - s0)), dg1 = d1 * uf.y * s1 * (1.f + gf.y * (1.f - s1));
                const float du0 = d0 * gf.x * s0, du1 = d1 * gf.y * s1;
                st32(sg + o, pack_bf16(dg0, dg1));
                st32(sg + kSlotBytes + o, pack_bf16(du0, du1));
              }
            }
            step_end();
            if (leader) {
              tma_store_2d(&em.c, sg, f0, row0);
              tma_store_2d(&em.c, sg + kSlotBytes, FF + f0, row0);
              bulk_commit();
              if (l_tile < num_tiles) {  // the pair is read out: it takes the boxes of the step two ahead
                bulk_wait_read<0>();
                aux_issue();
              }
            }
            ++ostep;
          }
        } else if (IO == 0 && p.c_fp32) {  // fp32 outputs and += are local-GEMM only
#pragma unroll
          for (int st = 0; st < TBN / 32; ++st) {  // 32 columns = 2 slots per step, double-buffered
            const int c0 = tn * TBN + 32 * st;
            if (c0 >= p.N) break;
            uint8_t* sb = slots + (ostep & 1) * (2 * kSlotBytes);
            step_begin(false);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * st + jj;
#pragma unroll
              for (int h = 0; h < 2; ++h)
                *reinterpret_cast<float2*>(sb + (jj >> 1) * kSlotBytes + off32(jj & 1, h)) =
                    make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
            step_end();
            if (leader) {
              // += (unsplit or split-K): the TMA unit adds the slot into C in the L2, one fp32 add per element
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                if (c0 + 16 * i >= p.N) break;
                if (p.accumulate) tma_reduce_add_2d(&em.c, sb + i * kSlotBytes, c0 + 16 * i, row0);
                else tma_store_2d(&em.c, sb + i * kSlotBytes, c0 + 16 * i, row0);
              }
              bulk_commit();
            }
            ++ostep;
          }
        } else {
          // RoPE: the position of each of this thread's two rows is fixed for the tile; TBN is a multiple of rope_D
          int rope_row[2] = {0, 0};
          if (EPI == 1) {
            rope_row[0] = (r0 % p.epi.rope_S) * (p.epi.rope_D >> 1);
            rope_row[1] = ((r0 + 8) % p.epi.rope_S) * (p.epi.rope_D >> 1);
          }
#pragma unroll
          for (int st = 0; st < TBN / 64; ++st) {  // 64 columns = 2 slots per step, double-buffered
            const int c0 = tn * TBN + 64 * st;
            if (c0 >= p.N) break;
            uint8_t* sb = slots + (ostep & 1) * (2 * kSlotBytes);
            const bool rot = EPI == 1 && c0 < p.epi.rope_cols;  // rope_cols is a multiple of rope_D (64 | 128)
            step_begin(false);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * st + jj;
              const int c = tn * TBN + 8 * j + cq;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                if (rot) {  // Q/K head columns: rotate the interleaved pair in registers
                  const int ti = rope_row[h] + (((8 * j + cq) & (p.epi.rope_D - 1)) >> 1);
                  const float cs = __ldg(p.epi.rope_cos + ti), sn = __ldg(p.epi.rope_sin + ti);
                  const float a = v0, b = v1;
                  v0 = a * cs - b * sn;
                  v1 = a * sn + b * cs;
                }
                if (IO == 0 && EPI == 0 && p.accumulate && r0 + 8 * h < p.M && c < p.N) {  // bf16 += (local, plain): one rounding
                  const float2 o =
                      __bfloat1622float2(*(reinterpret_cast<const __nv_bfloat162*>(p.C) + ((int64_t)(r0 + 8 * h) * p.ldc + c) / 2));
                  v0 += o.x;
                  v1 += o.y;
                }
                st32(sb + (jj >> 2) * kSlotBytes + off16(jj & 3, h), pack_bf16(v0, v1));
              }
            }
            step_end();
            if (leader) {
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                if (c0 + 32 * i >= p.N) break;
                tma_store_2d(&em.c, sb + i * kSlotBytes, c0 + 32 * i, row0);
              }
              bulk_commit();
            }
            ++ostep;
          }
        }
      } else {
        // reduce-scatter: add each fp32 pair into the buffer of the rank that owns the row (peer-mapped)
#pragma unroll
        for (int j = 0; j < TBN / 8; ++j) {
          const int c = tn * TBN + 8 * j + cq;
          if (c >= p.N) continue;  // N is even: c < N ⇒ c + 1 < N
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
            if (r >= p.M) continue;
            const int owner = r / pm.rows_per_rank;
            float* dst = pm.c[owner] + (int64_t)(r - owner * pm.rows_per_rank) * p.ldc + c;
            atomicAdd(dst, acc[4 * j + 2 * h]);
            atomicAdd(dst + 1, acc[4 * j + 2 * h + 1]);
          }
        }
      }
    }
    if (IO != 2 && leader) bulk_wait_all();  // the last stores have left shared memory
    if (IO == 2) __threadfence_system();  // peer reductions are performed before this kernel retires (a barrier follows)
  }
}

// ---------------------------------------------------------------- host side
int g_num_sms = 0;

// Split-K for reduce-add outputs: for grids that already fill the machine, splitting K to smooth wave quantisation costs more
// in extra fp32 reductions than the idle tail saves, so the automatic policy only splits when the output has fewer than half as
// many tiles as there are CTAs, i.e. when most SMs would otherwise sit idle for the whole kernel; slices keep >= 16 k-blocks
// (K >= 1024) each.
int choose_split_k(int tiles, int units, int num_kb) {
  if (tiles * 2 > units) return 1;
  int s = units / tiles;
  if (s > 8) s = 8;
  while (s > 1 && num_kb / s < 16) --s;
  return s < 1 ? 1 : s;
}

int g_split_k_mode = -1;  // -1 auto, 0/1 off, n>1 forced

const GemmEpilogue kPlain = {};

template <int A_MN, int B_MN, int EPI, int IO, int TBN>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream, const EpiMaps* emp,
           const PeerMaps* pmp, const CUtensorMap* tgp, const CUtensorMap* tg2p) {
  static const EpiMaps kNoEpi = {};
  static const PeerMaps kNoPeers = {};
  const EpiMaps& em = emp ? *emp : kNoEpi;
  const PeerMaps& pm = pmp ? *pmp : kNoPeers;
  const CUtensorMap& tg = tgp ? *tgp : ta;
  const CUtensorMap& tg2 = tg2p ? *tg2p : tg;
  using G = Geo<IO, TBN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_kernel<A_MN, B_MN, EPI, IO, TBN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)G::kSmemBytes);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  if (g_num_sms == 0) g_num_sms = pbhost::num_sms();
  int grid = g_num_sms;
  const int tiles_n = EPI == 2 ? (p.swiglu_ff + TBN / 2 - 1) / (TBN / 2) : (p.N + TBN - 1) / TBN;
  const int tiles = ((p.M + BM - 1) / BM) * tiles_n * p.split_k;
  // IO = 1 / 3 need every CTA resident at once (tiles wait on flags other CTAs publish): the grid never exceeds the SM count
  if (tiles < grid) grid = tiles;
  gemm_bf16_kernel<A_MN, B_MN, EPI, IO, TBN><<<grid, kThreads, G::kSmemBytes, stream>>>(ta, tb, tg, tg2, p, em, pm);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : (int)e;
}

constexpr int variant(int io, int epi, int a_mn, int b_mn, int wide) { return wide << 6 | io << 4 | epi << 2 | a_mn << 1 | b_mn; }

// (I/O mode, epilogue, operand layouts, tile width) → kernel. These 23 instantiations are all the entry points accept: every
// layout for the plain local GEMM, RoPE / SwiGLU on K-major B, SwiGLU backward on MN-major B, each in both tile widths, and
// K-major A for the collective modes (narrow tiles only).
int dispatch(int io, int epi, const GemmParams& p, const CUtensorMap& ta, const CUtensorMap& tb, cudaStream_t stream,
             const EpiMaps* em, const PeerMaps* pm = nullptr, const CUtensorMap* tg = nullptr, const CUtensorMap* tg2 = nullptr,
             bool wide = false) {
  switch (variant(io, epi, p.a_mn, p.b_mn, wide)) {
#define PB_GEMM_VARIANT(IO, EPI, A_MN, B_MN, TBN)         \
  case variant(IO, EPI, A_MN, B_MN, TBN == kWideBN):      \
    return launch<A_MN, B_MN, EPI, IO, TBN>(ta, tb, p, stream, em, pm, tg, tg2);
    PB_GEMM_VARIANT(0, 0, 0, 0, BN)
    PB_GEMM_VARIANT(0, 0, 0, 1, BN)
    PB_GEMM_VARIANT(0, 0, 1, 0, BN)
    PB_GEMM_VARIANT(0, 0, 1, 1, BN)
    PB_GEMM_VARIANT(0, 1, 0, 0, BN)
    PB_GEMM_VARIANT(0, 2, 0, 0, BN)
    PB_GEMM_VARIANT(0, 3, 0, 1, BN)
    PB_GEMM_VARIANT(0, 0, 0, 0, kWideBN)
    PB_GEMM_VARIANT(0, 0, 0, 1, kWideBN)
    PB_GEMM_VARIANT(0, 0, 1, 0, kWideBN)
    PB_GEMM_VARIANT(0, 0, 1, 1, kWideBN)
    PB_GEMM_VARIANT(0, 1, 0, 0, kWideBN)
    PB_GEMM_VARIANT(0, 2, 0, 0, kWideBN)
    PB_GEMM_VARIANT(0, 3, 0, 1, kWideBN)
    PB_GEMM_VARIANT(1, 0, 0, 0, BN)
    PB_GEMM_VARIANT(1, 0, 0, 1, BN)
    PB_GEMM_VARIANT(2, 0, 0, 0, BN)
    PB_GEMM_VARIANT(2, 0, 0, 1, BN)
    PB_GEMM_VARIANT(3, 0, 0, 0, BN)
    PB_GEMM_VARIANT(3, 0, 0, 1, BN)
    PB_GEMM_VARIANT(3, 1, 0, 0, BN)
    PB_GEMM_VARIANT(3, 2, 0, 0, BN)
    PB_GEMM_VARIANT(3, 3, 0, 1, BN)
#undef PB_GEMM_VARIANT
    default:
      return -7;
  }
}

int g_tile_mode = -1;  // -1 automatic (tile_policy), BN or kWideBN forced

// Split-K slices of an fp32 reduce-add output under the current split mode, for a grid of `tiles` output tiles.
int split_for(int tiles, int num_kb) {
  if (g_split_k_mode == 0 || g_split_k_mode == 1) return 1;
  if (g_split_k_mode > 1) return num_kb / g_split_k_mode >= 1 ? g_split_k_mode : 1;
  if (g_num_sms == 0) g_num_sms = pbhost::num_sms();
  return choose_split_k(tiles, g_num_sms > 0 ? g_num_sms : 1, num_kb);
}

// Tile width of a local GEMM, from the shape alone. A wide tile does the work of two narrow ones per pass over its k-blocks and
// brings 48 KB per k-block instead of 2 x 32 KB, so it runs kWideGainPct % more FLOP per unit of time. The persistent grid runs
// ceil(tiles / SMs) rounds of equal tiles; the wide tile is taken when its rounds, each twice as long, net of that gain, take no
// longer than the narrow rounds. Narrow stays for M <= 128 (one row of tiles: the decode-step GEMMs), and for fp32 reduce-add
// outputs that split K under either width (a split sums through atomics, so a different width would change the result).
constexpr int kWideGainPct = 10;
int tile_policy(int M, int N, int K, int epi, int c_fp32, int accumulate, int units) {
  if (M <= BM) return BN;
  const int tm = (M + BM - 1) / BM;
  const int t128 = tm * (epi == 2 ? (N / 2 + 63) / 64 : (N + BN - 1) / BN);
  const int t256 = tm * (epi == 2 ? (N / 2 + 127) / 128 : (N + kWideBN - 1) / kWideBN);
  if (c_fp32 && accumulate) {
    const int num_kb = (K + BK - 1) / BK;
    if (choose_split_k(t128, units, num_kb) > 1 || choose_split_k(t256, units, num_kb) > 1) return BN;
  }
  const int r128 = (t128 + units - 1) / units, r256 = (t256 + units - 1) / units;
  return 2 * r256 * 100 <= r128 * (100 + kWideGainPct) ? kWideBN : BN;
}

// Argument rules of the fused epilogues, for both entry points; N is the N of the product A·Bᵀ (2·FF for SwiGLU, FF for SwiGLU
// backward). -7: the epilogue does not exist for this layout / output; -3 / -4: RoPE tables / geometry; -5: SwiGLU geometry.
int check_epilogue(const GemmEpilogue& e, int M, int N, int a_mn, int b_mn, int c_fp32, int accumulate) {
  if (e.kind == 0) return 0;
  if (e.kind < 0 || e.kind > 3 || a_mn || b_mn != (e.kind == 3) || c_fp32 || accumulate) return -7;
  if (e.kind == 1) {
    if (e.rope_cos == nullptr || e.rope_sin == nullptr || e.rope_S <= 0 || M % e.rope_S != 0) return -3;
    if ((e.rope_D != 64 && e.rope_D != 128) || e.rope_cols % e.rope_D != 0 || e.rope_cols > N) return -4;
    return 0;
  }
  // a tile covers 64 features; aux is the base of a TMA map (epilogue_maps): 16-byte aligned address and row stride
  if (N % (e.kind == 2 ? 128 : 64) != 0 || e.aux == nullptr || (e.ld_aux % 8) || (reinterpret_cast<uintptr_t>(e.aux) & 15)) return -5;
  if (e.kind == 3 && M <= BM) return -5;
  return 0;
}

GemmParams make_params(void* C, int M, int N, int K, int ldc, int a_mn, int b_mn, int c_fp32, int accumulate, const GemmEpilogue& e) {
  GemmParams p = {};
  p.M = M;
  p.N = N;
  p.K = K;
  p.ldc = ldc;
  p.a_mn = a_mn != 0;
  p.b_mn = b_mn != 0;
  p.c_fp32 = c_fp32;
  p.accumulate = accumulate;
  p.split_k = 1;
  p.C = C;
  p.epi = e;
  p.swiglu_ff = e.kind == 2 ? N / 2 : e.kind == 3 ? N : 0;
  return p;
}

// A / B operand tensor maps: K-major {64 k, rows} boxes, MN-major {64 mn, 64 k} boxes.
int operand_tmap(CUtensorMap* m, const void* ptr, int mn, int K, int ld, int mn_major, int box_rows) {
  return mn_major ? pbhost::cached_tmap(m, ptr, (uint64_t)K, (uint64_t)mn, (uint64_t)ld, 64, BK)
                  : pbhost::cached_tmap(m, ptr, (uint64_t)mn, (uint64_t)K, (uint64_t)ld, BK, box_rows);
}

// The staged epilogue's maps (the entry points' checks and check_epilogue give TMA its 16-byte aligned addresses and row
// strides): C [M, N] (SwiGLU backward: d_gate_up [M, 2·N]), h [M, FF] for SwiGLU, the saved gate_up [M, 2·N] for SwiGLU backward.
int epilogue_maps(EpiMaps* em, void* C, int M, int N, int ldc, int c_fp32, const GemmEpilogue& e) {
  int rc;
  if ((rc = pbhost::cached_tmap_staging(&em->c, C, M, e.kind == 3 ? 2 * N : N, ldc, c_fp32 != 0))) return rc;
  if (e.kind == 2 && (rc = pbhost::cached_tmap_staging(&em->h, e.aux, M, N / 2, e.ld_aux, false))) return rc;
  if (e.kind == 3 && (rc = pbhost::cached_tmap_staging(&em->gu, e.aux, M, 2 * N, e.ld_aux, false))) return rc;
  return 0;
}

}  // namespace

// Split-K policy for fp32 reduce-add outputs: -1 = automatic (default), 0 = never, n > 1 = always n slices (testing).
PB_EXPORT int pb_gemm_set_split_k(int mode) {
  const int old = g_split_k_mode;
  g_split_k_mode = mode;
  return old;
}

// Tile width of pb_gemm_bf16: -1 = automatic (default, tile_policy), 128 or 256 = always that width (testing). Returns the old
// mode; -9 and no change for any other value.
PB_EXPORT int pb_gemm_set_tile(int mode) {
  if (mode != -1 && mode != BN && mode != kWideBN) return -9;
  const int old = g_tile_mode;
  g_tile_mode = mode;
  return old;
}

// The tile width (128 | 256) the automatic policy gives pb_gemm_bf16 for this shape on a GPU with `num_sms` SMs; host only.
PB_EXPORT int pb_gemm_tile_policy(int M, int N, int K, int epi_kind, int c_fp32, int accumulate, int num_sms) {
  return tile_policy(M, N, K, epi_kind, c_fp32, accumulate, num_sms > 0 ? num_sms : 1);
}

// C[M, N] (bf16 | fp32, += with `accumulate`) = A·Bᵀ, optionally with a fused epilogue (null `epi` = plain).
// lda/ldb: row stride (elements) of the matrix AS STORED (see header comment).
//   RoPE:            y = x·Wᵀ with the Q/K head columns rotated (the fused QKV projection)
//   SwiGLU:          gate_up = x·W13ᵀ [M, N = 2·FF] with W13 = [gate rows | up rows] into C, and h = silu(gate)·up into epi->aux
//   SwiGLU backward: dh = dy·W2 [M, N = FF] never leaves registers: C = d_gate_up [M, 2·FF] from dh and the saved gate_up (epi->aux)
// RoPE and SwiGLU take K-major operands, SwiGLU backward K-major A and MN-major B; all three write bf16 without accumulating.
PB_EXPORT int pb_gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc, int a_mn_major,
                           int b_mn_major, int c_fp32, int accumulate, const GemmEpilogue* epi, cudaStream_t stream) {
  const GemmEpilogue& e = epi ? *epi : kPlain;
  int rc;
  if ((rc = check_epilogue(e, M, N, a_mn_major, b_mn_major, c_fp32, accumulate))) return rc;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((lda % 8) || (ldb % 8) || (ldc % (c_fp32 ? 4 : 8))) return -1;
  if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) | reinterpret_cast<uintptr_t>(C)) & 15) return -2;
  if (g_num_sms == 0) g_num_sms = pbhost::num_sms();
  const int tbn = g_tile_mode > 0 ? g_tile_mode : tile_policy(M, N, K, e.kind, c_fp32, accumulate, g_num_sms > 0 ? g_num_sms : 1);
  const bool wide = tbn == kWideBN;
  CUtensorMap ta, tb, tup;
  if ((rc = operand_tmap(&ta, A, M, K, lda, a_mn_major, BM))) return rc;
  if (wide && e.kind == 2) {  // SwiGLU: the gate rows and the up rows of W13 as two maps of FF rows each
    const int FF = N / 2;
    if ((rc = pbhost::cached_tmap(&tb, B, (uint64_t)FF, (uint64_t)K, (uint64_t)ldb, BK, 128))) return rc;
    const void* up = static_cast<const __nv_bfloat16*>(B) + (int64_t)FF * ldb;
    if ((rc = pbhost::cached_tmap(&tup, up, (uint64_t)FF, (uint64_t)K, (uint64_t)ldb, BK, 128))) return rc;
  } else if ((rc = operand_tmap(&tb, B, N, K, ldb, b_mn_major, e.kind == 2 ? 64 : tbn))) {
    return rc;
  }
  EpiMaps em = {};
  if ((rc = epilogue_maps(&em, C, M, N, ldc, c_fp32, e))) return rc;
  GemmParams p = make_params(C, M, N, K, ldc, a_mn_major, b_mn_major, c_fp32, accumulate, e);
  if (c_fp32 && accumulate) p.split_k = split_for(((M + BM - 1) / BM) * ((N + tbn - 1) / tbn), (K + BK - 1) / BK);  // plain only
  return dispatch(0, e.kind, p, ta, tb, stream, &em, nullptr, wide && e.kind == 2 ? &tup : nullptr, nullptr, wide);
}

// ---------------------------------------------------------------------------------------------------------------------------
// all-gather ⊕ GEMM:  C[n·M_local, N] = [A_0; A_1; …; A_{n-1}] · Bᵀ, A_r = rank r's [M_local, K] block in the symmetric heap.
// a_peers[r] is the address of rank r's block AS MAPPED IN THIS PROCESS. The caller brackets the call with heap barriers (every
// rank's block written before, nobody overwrites it until all ranks are done). K-major A, bf16 output.
// a_full: local [n·M_local, K] bf16 scratch that receives the remote row blocks (by-product: the gathered A, minus the local block);
// flags: n·M_local/128 uint32 counters in local memory (zeroed here, on the stream).
// b_mn_major: B stored [K, N] (the transposed weight of a backward GEMM) instead of [N, K].
PB_EXPORT int pb_gemm_allgather(const void* const* a_peers, int n, int rank, const void* B, void* C, void* a_full, uint32_t* flags,
                                int M_local, int N, int K, int lda, int ldb, int ldc, int b_mn_major, cudaStream_t stream) {
  if (n < 1 || n > 8 || rank < 0 || rank >= n || M_local % BM != 0) return -6;
  if ((lda % 8) || (ldb % 8) || (ldc % 8) || (K % 8)) return -1;
  if (reinterpret_cast<uintptr_t>(C) & 15) return -2;
  PeerMaps pm = {};
  pm.n = n;
  pm.rows_per_rank = M_local;
  pm.rank = rank;
  pm.flags = flags;
  int rc;
  if (n > 1) {
    cudaError_t e = cudaMemsetAsync(flags, 0, sizeof(uint32_t) * (size_t)(n * (M_local / BM)), stream);
    if (e != cudaSuccess) return (int)e;
  }
  for (int r = 0; r < n; ++r)
    if ((rc = pbhost::cached_tmap(&pm.m[r], a_peers[r], (uint64_t)M_local, (uint64_t)K, (uint64_t)lda, BK, BM))) return rc;
  const int M = n * M_local;
  CUtensorMap tfull, tb;
  if ((rc = pbhost::cached_tmap(&tfull, a_full, (uint64_t)M, (uint64_t)K, (uint64_t)K, BK, BM))) return rc;
  if ((rc = operand_tmap(&tb, B, N, K, ldb, b_mn_major, BN))) return rc;
  EpiMaps em = {};
  if ((rc = epilogue_maps(&em, C, M, N, ldc, 0, kPlain))) return rc;
  return dispatch(1, 0, make_params(C, M, N, K, ldc, 0, b_mn_major, 0, 0, kPlain), tfull, tb, stream, &em, &pm);
}

// GEMM ⊕ reduce-scatter:  every rank holds a K-shard (A [M, K_local], B [N, K_local]); rank r ends up with rows
// [r·M/n, (r+1)·M/n) of Σ_ranks A·Bᵀ in its fp32 buffer c_peers[r] ([M/n, N], zeroed by the caller before the opening barrier).
PB_EXPORT int pb_gemm_reduce_scatter(const void* A, const void* B, float* const* c_peers, int n, int rank, int M, int N, int K, int lda,
                                     int ldb, int ldc, int b_mn_major, cudaStream_t stream) {
  if (n < 1 || n > 8 || rank < 0 || rank >= n || M % n != 0 || (M / n) % BM != 0) return -6;
  if ((lda % 8) || (ldb % 8) || (ldc % 4)) return -1;
  PeerMaps pm = {};
  pm.n = n;
  pm.rows_per_rank = M / n;
  pm.rank = rank;
  for (int r = 0; r < n; ++r) pm.c[r] = c_peers[r];
  int rc;
  CUtensorMap ta, tb;
  if ((rc = operand_tmap(&ta, A, M, K, lda, 0, BM))) return rc;
  if ((rc = operand_tmap(&tb, B, N, K, ldb, b_mn_major, BN))) return rc;
  return dispatch(2, 0, make_params(c_peers[rank], M, N, K, ldc, 0, b_mn_major, 1, 1, kPlain), ta, tb, stream, nullptr, &pm);
}

// ---------------------------------------------------------------------------------------------------------------------------
// parameter all-gather ⊕ GEMM (IO = 3; ZeRO-3 / train.reshard_after_forward): the weight W [rowsW, colsW] is sharded by rows
// over n ranks (rank r: rows [r·rowsW/n, (r+1)·rowsW/n) at w_peers[r], the address AS MAPPED IN THIS PROCESS). The kernel gathers
// it into w_full (local, [rowsW, colsW]) tile by tile WHILE it multiplies; no collective, no barrier (shards are read-only here).
//   b_mn_major = 0 (forward)        C[M, rowsW] = A[M, colsW] · Wᵀ          epilogue: plain | RoPE | SwiGLU (W = W13, N = 2·FF)
//   b_mn_major = 1 (input gradient) C[M, colsW] = A[M, rowsW] · W           epilogue: plain | SwiGLU backward (W = W2, N = FF)
// `epi` as for pb_gemm_bf16. flags: n·4 uint32 in local memory (zeroed here, on the stream). bf16 everywhere, M > 128.
// own_resident = 1: W is already complete in w_full (gathered ahead by the previous kernel): no gather, no gating.
// next_peers != nullptr: additionally gather the weight [next_rows, next_cols] (same n ranks) the NEXT GEMM will consume into
// next_full — un-gated, complete when this kernel retires.
PB_EXPORT int pb_gemm_wgather(const void* A, const void* const* w_peers, int n, int rank, void* w_full, uint32_t* flags, void* C, int M,
                              int rowsW, int colsW, int lda, int ldc, int b_mn_major, const GemmEpilogue* epi, int own_resident,
                              const void* const* next_peers, void* next_full, int next_rows, int next_cols, cudaStream_t stream) {
  const GemmEpilogue& e = epi ? *epi : kPlain;
  if (n < 1 || n > 8 || rank < 0 || rank >= n || rowsW % n != 0 || colsW % 64 != 0) return -6;
  if ((lda % 8) || (ldc % 8)) return -1;
  if (reinterpret_cast<uintptr_t>(C) & 15) return -2;
  const int N = b_mn_major ? colsW : rowsW, K = b_mn_major ? rowsW : colsW;
  int rc;
  if ((rc = check_epilogue(e, M, N, 0, b_mn_major, 0, 0))) return rc;
  if (M <= BM) return -8;  // training shapes only; tiny M goes through an explicit gather on the host side
  const int rpr = rowsW / n;
  PeerMaps pm = {};
  pm.n = n;
  pm.rows_per_rank = rpr;
  pm.rank = rank;
  pm.flags = flags;
  pm.cpr = (rpr + 127) / 128;
  pm.col_chunks = colsW / 64;
  pm.spc = (pm.cpr + kGatherSub - 1) / kGatherSub;
  pm.gate = own_resident ? 0 : 1;
  CUtensorMap tg2;
  bool have_next = false;
  if (next_peers != nullptr && next_full != nullptr && next_rows > 0) {
    if (next_rows % n != 0 || next_cols % 64 != 0) return -6;
    const int nrpr = next_rows / n;
    pm.nn = n;
    pm.ncpr = (nrpr + 127) / 128;
    pm.ncol_chunks = next_cols / 64;
    for (int t = 0; t < n; ++t) pm.norder[t] = (rank + 1 + t) % n;  // remote blocks first (they take longest), own block last
    for (int r = 0; r < n; ++r)
      if ((rc = pbhost::cached_tmap(&pm.nm[r], next_peers[r], (uint64_t)nrpr, (uint64_t)next_cols, (uint64_t)next_cols, BK, 128))) return rc;
    if ((rc = pbhost::cached_tmap_blocks(&tg2, next_full, (uint64_t)nrpr, (uint64_t)next_cols, (uint64_t)n, BK, 128))) return rc;
    have_next = true;
  }
  if (e.kind == 2 && n % 2 == 0) {
    // a tile needs gate rows (blocks < n/2) and the matching up rows (blocks >= n/2): fetch them pairwise, own pair first
    const int h = n / 2, g0 = rank % h;
    for (int t = 0; t < h; ++t) {
      const int g = (g0 + t) % h;
      pm.order[2 * t] = rank >= h ? g + h : g;
      pm.order[2 * t + 1] = rank >= h ? g : g + h;
    }
    pm.start = (g0 * rpr) / 64;  // tiles are 64 features wide
  } else {
    for (int t = 0; t < n; ++t) pm.order[t] = (rank + t) % n;
    if (e.kind == 2) pm.start = 0;
    else pm.start = b_mn_major ? (rank * rpr) / BK : (rank * rpr) / BN;
  }
  if (!own_resident) {
    cudaError_t err = cudaMemsetAsync(flags, 0, sizeof(uint32_t) * (size_t)(n * kGatherSub), stream);
    if (err != cudaSuccess) return (int)err;
  }
  for (int r = 0; r < n; ++r)
    if ((rc = pbhost::cached_tmap(&pm.m[r], w_peers[r], (uint64_t)rpr, (uint64_t)colsW, (uint64_t)colsW, BK, 128))) return rc;
  CUtensorMap tg, ta, tb;
  if ((rc = pbhost::cached_tmap_blocks(&tg, w_full, (uint64_t)rpr, (uint64_t)colsW, (uint64_t)n, BK, 128))) return rc;
  if ((rc = operand_tmap(&ta, A, M, K, lda, 0, BM))) return rc;
  if ((rc = operand_tmap(&tb, w_full, N, K, colsW, b_mn_major, e.kind == 2 ? 64 : BN))) return rc;
  EpiMaps em = {};
  if ((rc = epilogue_maps(&em, C, M, N, ldc, 0, e))) return rc;
  return dispatch(3, e.kind, make_params(C, M, N, K, ldc, 0, b_mn_major, 0, 0, e), ta, tb, stream, &em, &pm, &tg,
                  have_next ? &tg2 : nullptr);
}
