#include "tmap.h"

#include <cuda_runtime.h>

#include <mutex>
#include <unordered_map>

namespace pbhost {

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(sym);
  });
  return fn;
}

// rows x cols (cols contiguous) matrix with row stride ld (elements); box = box_cols x box_rows; esize 1 (fp8/bytes) | 2 (bf16) | 4 (f32)
// esize -4: rows of `cols` uint32 words, NO swizzle (MXFP8 scale-factor atoms: 128 words = 512 bytes per row)
static int make_tmap(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols,
                     uint32_t box_rows, int esize) {
  EncodeFn enc = get_encode();
  if (!enc) return -10;
  // Driver entry points need a current context on THIS thread; autograd's backward threads may not have
  // bound the primary context yet (seen as CUDA_ERROR_INVALID_CONTEXT). A no-op runtime call binds it.
  static thread_local bool ctx_bound = false;  // once per thread: cudaFree is illegal during graph capture
  if (!ctx_bound) {
    cudaFree(nullptr);
    ctx_bound = true;
  }
  cuuint64_t dims[2] = {cols, rows};
  const bool raw = esize == -4;
  if (raw) esize = 4;
  cuuint64_t strides[1] = {ld * (uint64_t)esize};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = raw ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = enc(map, dt, 2,
                   const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, raw ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -11 - (int)r;
}

// 3-D view of a bf16 [rows, cols] matrix as {64 columns, rows, cols/64 column chunks}: ONE box of {64, box_rows, chunks} lands in
// shared memory as `chunks` consecutive [box_rows x 128 B] 128B-swizzled blocks — the operand layout of the attention kernels —
// with a single cp.async.bulk.tensor.3d instead of one 2-D box per 64-column chunk.
static int make_tmap3(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, uint32_t chunks) {
  EncodeFn enc = get_encode();
  if (!enc) return -10;
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(nullptr);
    ctx_bound = true;
  }
  cuuint64_t dims[3] = {64, rows, cols / 64};
  cuuint64_t strides[2] = {ld * 2, 128};
  cuuint32_t box[3] = {64, box_rows, chunks};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -11 - (int)r;
}

struct MapKey {
  const void* ptr;
  uint64_t rows, cols, ld;
  uint32_t bc, br;
  int esize;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && bc == o.bc && br == o.br && esize == o.esize;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    auto mix = [&](uint64_t v) { h ^= std::hash<uint64_t>()(v) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
    mix(k.rows), mix(k.cols), mix(k.ld), mix(k.bc), mix(k.br), mix((uint64_t)k.esize);
    return h;
  }
};

int cached_tmap(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t bc, uint32_t br,
                int esize) {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  MapKey key{ptr, rows, cols, ld, bc, br, esize};
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it == cache.end()) {
    CUtensorMap m;
    int rc = make_tmap(&m, ptr, rows, cols, ld, bc, br, esize);
    if (rc) return rc;
    if (cache.size() > 8192) cache.clear();
    it = cache.emplace(key, m).first;
  }
  *out = it->second;
  return 0;
}


int cached_tmap3(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, uint32_t chunks) {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  MapKey key{ptr, rows, cols, ld, chunks, box_rows, 33};
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it == cache.end()) {
    CUtensorMap m;
    int rc = make_tmap3(&m, ptr, rows, cols, ld, box_rows, chunks);
    if (rc) return rc;
    if (cache.size() > 8192) cache.clear();
    it = cache.emplace(key, m).first;
  }
  *out = it->second;
  return 0;
}

// [blocks][rows][cols] bf16 (dense: block stride = rows*cols) with boxes of {box_cols, box_rows, 1}: a box never crosses a block, rows
// past the end of a block are clipped on stores / zero-filled on loads (the weight-gather copier of gemm_sm90.cu relies on that).
int cached_tmap_blocks(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t blocks, uint32_t box_cols, uint32_t box_rows) {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  MapKey key{ptr, rows, cols, blocks, box_cols, box_rows, 34};
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it == cache.end()) {
    EncodeFn enc = get_encode();
    if (!enc) return -10;
    static thread_local bool ctx_bound = false;
    if (!ctx_bound) {
      cudaFree(nullptr);
      ctx_bound = true;
    }
    CUtensorMap m;
    cuuint64_t dims[3] = {cols, rows, blocks};
    cuuint64_t strides[2] = {cols * 2, rows * cols * 2};
    cuuint32_t box[3] = {box_cols, box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return -11 - (int)r;
    if (cache.size() > 8192) cache.clear();
    it = cache.emplace(key, m).first;
  }
  *out = it->second;
  return 0;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

}  // namespace pbhost
