#include "tmap.h"

#include <cuda_runtime.h>

#include <mutex>
#include <unordered_map>

namespace pbhost {
namespace {

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

// `ld` is the row stride of a 2-D map and the block count of a blocks view
struct MapKey {
  const void* ptr;
  uint64_t rows, cols, ld;
  uint32_t bc, br;
  bool blocks;
  CUtensorMapDataType dtype;
  CUtensorMapSwizzle swizzle;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && bc == o.bc && br == o.br && blocks == o.blocks &&
           dtype == o.dtype && swizzle == o.swizzle;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    auto mix = [&](uint64_t v) { h ^= std::hash<uint64_t>()(v) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
    mix(k.rows), mix(k.cols), mix(k.ld), mix(k.bc), mix(k.br), mix((uint64_t)k.blocks);
    mix((uint64_t)k.dtype), mix((uint64_t)k.swizzle);
    return h;
  }
};

// Encode (once per key) a map of `rank` dimensions with the key's element type and swizzle.
int cached(CUtensorMap* out, const MapKey& key, cuuint32_t rank, const cuuint64_t* dims, const cuuint64_t* strides,
           const cuuint32_t* box) {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it == cache.end()) {
    EncodeFn enc = get_encode();
    if (!enc) return -10;
    // Driver entry points need a current context on THIS thread; autograd's backward threads may not have
    // bound the primary context yet (seen as CUDA_ERROR_INVALID_CONTEXT). A no-op runtime call binds it.
    static thread_local bool ctx_bound = false;  // once per thread: cudaFree is illegal during graph capture
    if (!ctx_bound) {
      cudaFree(nullptr);
      ctx_bound = true;
    }
    const cuuint32_t estr[3] = {1, 1, 1};
    CUtensorMap m;
    CUresult r = enc(&m, key.dtype, rank, const_cast<void*>(key.ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, key.swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return -11 - (int)r;
    if (cache.size() > 8192) cache.clear();
    it = cache.emplace(key, m).first;
  }
  *out = it->second;
  return 0;
}

}  // namespace

int cached_tmap(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols, uint32_t box_rows) {
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {ld * 2};
  const cuuint32_t box[2] = {box_cols, box_rows};
  return cached(out, {ptr, rows, cols, ld, box_cols, box_rows, false, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B}, 2,
                dims, strides, box);
}

int cached_tmap_staging(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, bool fp32) {
  const uint64_t esz = fp32 ? 4 : 2;
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {ld * esz};
  const cuuint32_t box[2] = {(cuuint32_t)(64 / esz), 64};
  const CUtensorMapDataType dt = fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  return cached(out, {ptr, rows, cols, ld, box[0], box[1], false, dt, CU_TENSOR_MAP_SWIZZLE_64B}, 2, dims, strides, box);
}

// A box never crosses a block: rows past the end of a block are clipped on stores / zero-filled on loads (the weight-gather
// copier of gemm_sm90.cu relies on that).
int cached_tmap_blocks(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t blocks, uint32_t box_cols,
                       uint32_t box_rows) {
  const cuuint64_t dims[3] = {cols, rows, blocks};
  const cuuint64_t strides[2] = {cols * 2, rows * cols * 2};
  const cuuint32_t box[3] = {box_cols, box_rows, 1};
  return cached(out, {ptr, rows, cols, blocks, box_cols, box_rows, true, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, CU_TENSOR_MAP_SWIZZLE_128B},
                3, dims, strides, box);
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
