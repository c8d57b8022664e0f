// Host-side construction of TMA tensor maps.  cuTensorMapEncodeTiled is resolved through the runtime
// (cudaGetDriverEntryPoint) so that the library does not link against libcuda.
#include <mutex>

#include "common.cuh"
#include "wgmma.cuh"

namespace hstu {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_rows_heads(CUtensorMap* out, const void* base, long long rows, int heads, int d, long long row_stride,
                         long long head_stride, int box_cols, int box_rows, int elem_bytes) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled is not available from this driver");
    return HSTU_ERR_CUDA;
  }
  if (elem_bytes != 1 && elem_bytes != 2) {
    set_error("tensor map: unsupported element size %d", elem_bytes);
    return HSTU_ERR_UNSUPPORTED;
  }
  const int sw_bytes = box_cols * elem_bytes;
  CUtensorMapSwizzle sw = sw_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : sw_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                          : sw_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                           : CU_TENSOR_MAP_SWIZZLE_NONE;
  if (sw == CU_TENSOR_MAP_SWIZZLE_NONE) {
    set_error("tensor map: unsupported box width %d", box_cols);
    return HSTU_ERR_UNSUPPORTED;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || ((row_stride * elem_bytes) & 15) || ((head_stride * elem_bytes) & 15)) {
    set_error("tensor map: base / strides must be 16-byte aligned (base=%p row_stride=%lld head_stride=%lld elements of %d bytes)",
              base, row_stride, head_stride, elem_bytes);
    return HSTU_ERR_UNSUPPORTED;
  }
  cuuint64_t dims[3] = {(cuuint64_t)d, (cuuint64_t)heads, (cuuint64_t)rows};
  cuuint64_t strides[2] = {(cuuint64_t)head_stride * elem_bytes, (cuuint64_t)row_stride * elem_bytes};
  if (heads == 1) strides[0] = (cuuint64_t)d * elem_bytes;  // unused dimension: any legal multiple of 16
  cuuint32_t box[3] = {(cuuint32_t)box_cols, 1u, (cuuint32_t)box_rows};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  // the maps only move bytes (no conversion, no OOB NaN fill), so one data type per element size will do
  const CUtensorMapDataType ty = elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = enc(out, ty, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%lld heads=%d d=%d row_stride=%lld head_stride=%lld box=%dx%d)",
              (int)r, rows, heads, d, row_stride, head_stride, box_cols, box_rows);
    return HSTU_ERR_CUDA;
  }
  return 0;
}

}  // namespace hstu
