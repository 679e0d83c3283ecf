// Host-side TMA tensor-map construction (driver entry point fetched through the runtime, so
// the extension does not link libcuda directly).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace dfno {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !ptr) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

// 2-D bf16 tensor map: inner dim = K elements (contiguous), outer = rows with pitch ld elements.
inline int make_map_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t rows, uint64_t ld_elems,
                       uint32_t box_inner, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return -1;
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

// 3-D bf16 tensor map (innermost first): dims (d0, d1, d2), element strides of d1 and d2, box (b0, b1, b2).
// SWIZZLE_128B: b0 * 2 bytes must be <= 128.  Loads zero-fill outside the tensor, stores are clipped.
inline int make_map_3d(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1_elems,
                       uint64_t s2_elems, uint32_t b0, uint32_t b1, uint32_t b2) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return -1;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {s1_elems * 2, s2_elems * 2};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

// rank-N (<= 5) bf16 tensor map, innermost dimension first: used for stores whose staging buffer is written with word
// stores.  `strides` (elements) belong to dims 1..rank-1 and must be multiples of 8; box[0] * 2 bytes must be a
// multiple of 16 and, with a swizzle, at most its span (32 / 64 / 128 B).  Stores are clipped at the extents.
inline int make_map_nd(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                       const uint32_t* box, CUtensorMapSwizzle swizzle) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc || rank < 1 || rank > 5) return -1;
  cuuint64_t d[5], st[4];
  cuuint32_t b[5], estr[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; estr[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) st[i] = strides[i] * 2;
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base), d, st, b,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

}  // namespace dfno
