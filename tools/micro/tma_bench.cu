// TMA delivery rate per SM as a function of box geometry, ring depth and row pitch: one CTA per SM, one thread issues 2-D tiled
// loads (SWIZZLE_128B, 64 bf16 = 128 B wide boxes) into a ring of 32 KB "tiles" and waits for each tile in order.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/tma_bench tools/micro/tma_bench.cu -lcuda
// Run  : tools/micro/tma_bench            → one JSON line per configuration (bytes per clock per SM, clocks per 32 KB tile)
#include <cstdio>
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

struct Cfg {
  int box_rows;     // rows per TMA box (64 | 128)
  int stages;       // tiles in flight
  int tiles;        // tiles per CTA
  int col_stride;   // columns between the boxes of one tile (interleaves several column offsets like K | V)
  int rows_per_cta; // row range each CTA walks (wraps)
};

__global__ void __launch_bounds__(64, 1) tma_kernel(const __grid_constant__ CUtensorMap map, Cfg c, unsigned long long* out) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ uint64_t full[8];
  const int boxes = 32768 / (c.box_rows * 128);
  if (threadIdx.x == 0) {
    for (int i = 0; i < 8; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(&full[i])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int row_base = ((int)blockIdx.x & 15) * 1024;  // 16 'batch elements' of 1024 rows, each shared by ~9 CTAs (as the q blocks of a head)
  const int row_mask = c.rows_per_cta - 1;             // power of two: no divisions in the issue path
  const int half_boxes = boxes > 1 ? boxes >> 1 : 1;
  const uint32_t smem0 = s32(smem);
  auto issue = [&](int t, int st) {
    const uint32_t bar = s32(&full[st]);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(32768u) : "memory");
    uint32_t dst = smem0 + st * 32768;
    for (int b = 0; b < boxes; ++b, dst += c.box_rows * 128) {
      // first half of the boxes: consecutive row groups at column 0, second half: the same rows at a second column offset (K | V)
      const int second = (boxes > 1 && b >= half_boxes) ? 1 : 0;
      const int rb = second ? b - half_boxes : b;
      const int row = row_base + (((t * half_boxes + rb) * c.box_rows) & row_mask);
      const int col = second * c.col_stride;
      asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
                   "l"(&map), "r"(bar), "r"(col), "r"(row)
                   : "memory");
    }
  };
  const long long t0 = clock64();
  int ist = 0;
  for (int t = 0; t < c.stages && t < c.tiles; ++t) {
    issue(t, ist);
    if (++ist == c.stages) ist = 0;
  }
  int st = 0;
  uint32_t ph = 0;
  for (int t = 0; t < c.tiles; ++t) {
    uint32_t ok = 0;
    while (!ok)
      asm volatile("{.reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p;}" : "=r"(ok) : "r"(s32(&full[st])), "r"(ph) : "memory");
    if (t + c.stages < c.tiles) issue(t + c.stages, st);
    if (++st == c.stages) st = 0, ph ^= 1;
  }
  out[blockIdx.x] = (unsigned long long)(clock64() - t0);
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                             const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
  void* sym = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaFree(nullptr);
  cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q);
  EncodeFn enc = (EncodeFn)sym;
  const uint64_t rows = 16384;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  unsigned long long* out;
  cudaMalloc(&out, sizeof(unsigned long long) * 256);
  cudaFuncSetAttribute(tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 6 * 32768);
  for (uint64_t cols : {2048ull, 6144ull}) {
    void* buf;
    cudaMalloc(&buf, rows * cols * 2);
    cudaMemset(buf, 1, rows * cols * 2);
    for (int promo = 0; promo < 2; ++promo)
      for (int box_rows : {64, 128})
        for (int stages : {2, 4, 6})
          for (int rows_per_cta : {1024, 110}) {  // 110 rows x 132 CTAs: everything L2-resident and reused
            CUtensorMap map;
            cuuint64_t dims[2] = {cols, rows};
            cuuint64_t strides[1] = {cols * 2};
            cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
            cuuint32_t es[2] = {1, 1};
            CUresult r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, buf, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_128B, promo ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_NONE,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) {
              printf("{\"error\": %d}\n", (int)r);
              continue;
            }
            Cfg c{box_rows, stages, 128, 1024, rows_per_cta == 110 ? 128 : 1024};  // 128: wraps inside 128 rows → L2 hits after the first pass
            for (int rep = 0; rep < 2; ++rep) tma_kernel<<<sms, 64, stages * 32768, 0>>>(map, c, out);
            cudaError_t e = cudaDeviceSynchronize();
            unsigned long long h[256];
            cudaMemcpy(h, out, sizeof(unsigned long long) * sms, cudaMemcpyDeviceToHost);
            unsigned long long mx = 0;
            for (int i = 0; i < sms; ++i) mx = h[i] > mx ? h[i] : mx;
            printf("{\"cols\": %llu, \"l2_promotion_256B\": %d, \"box_rows\": %d, \"stages\": %d, \"rows_per_cta\": %d, \"clk_per_32KB_tile\": %.0f, "
                   "\"bytes_per_clk_per_sm\": %.1f, \"err\": %d}\n",
                   (unsigned long long)cols, promo, box_rows, stages, c.rows_per_cta, (double)mx / c.tiles, 32768.0 * c.tiles / (double)mx, (int)e);
          }
    cudaFree(buf);
  }
  return 0;
}
