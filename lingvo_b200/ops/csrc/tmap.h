// TMA tensor maps shared by the GEMM and the flash attention (defined in gemm_wgmma.cu).
#pragma once

#include <cuda.h>

#include <cstdint>

namespace lb {

// 3-D map over a [groups, rows, inner] view (strides in elements); box = [1, box_rows,
// 128 bytes], 128B swizzle. Binds the device's primary context to the calling thread
// first, since the encoder is a driver call.
CUtensorMap MakeMap(const void* base, int64_t inner, int64_t rows, int64_t groups,
                    int64_t row_stride, int64_t group_stride, int box_rows,
                    CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, int elem_bytes = 2);

}  // namespace lb
