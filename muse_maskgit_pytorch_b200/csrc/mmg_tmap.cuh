// Host-side TMA descriptor construction shared by the GEMM and attention launchers.
#pragma once
#include "mmg_common.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <mutex>

namespace mmg {

// ------------------------------------------------------------------------------------------------------------------
// cuTensorMapEncodeTiled through the runtime's driver entry point (libmmg.so does not link libcuda directly, so it
// can be dlopen'ed on a machine without a driver for the symbol-export test).
// ------------------------------------------------------------------------------------------------------------------
inline PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr; cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
  });
  return fn;
}

// tensor map, rank <= 4, innermost dim contiguous, 128B swizzle, zero OOB fill (loads) / OOB elements skipped (stores, reductions).
inline int make_tmap(CUtensorMap* m, CUtensorMapDataType dt, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes /*rank-1*/,
                     const uint32_t* box);
inline int make_tmap_bf16(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box);
}
inline int make_tmap_u8(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, rank, dims, strides_bytes, box);     // e4m3 operands: TMA moves bytes
}
inline int make_tmap_f32(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, rank, dims, strides_bytes, box);
}
inline int make_tmap(CUtensorMap* m, CUtensorMapDataType dt, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes /*rank-1*/,
                     const uint32_t* box) {
  auto enc = get_encode();
  if (!enc) return fail(MMG_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gd[5]; cuuint64_t gs[4]; cuuint32_t bx[5]; cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
  CUresult r = enc(m, dt, rank, const_cast<void*>(base), gd, gs, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MMG_ECUDA, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dims %llu x %llu, box %u x %u)",
                                     (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
  return MMG_OK;
}


}  // namespace mmg
