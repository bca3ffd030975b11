// Host-side TMA tensor-map construction (cuTensorMapEncodeTiled through the runtime's driver entry point) with a
// process-wide cache keyed by (pointer, shape, stride, box, element type, swizzle); 0 = success.
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace pbhost {
// rows x cols matrix (cols contiguous), row stride `ld` elements, boxes of box_cols x box_rows.
// bf16, 128B-swizzled boxes of box_cols x box_rows.
int cached_tmap(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols, uint32_t box_rows);
// bf16 or fp32, 64B-swizzled boxes of 64 rows x 64 bytes: the epilogue staging slots of the local GEMM (gemm_sm90.cu).
int cached_tmap_staging(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, bool fp32);
// dense [blocks][rows][cols] view, boxes {box_cols, box_rows, 1} (rows clipped per block)
int cached_tmap_blocks(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t cols, uint64_t blocks, uint32_t box_cols, uint32_t box_rows);
int num_sms();
}  // namespace pbhost
