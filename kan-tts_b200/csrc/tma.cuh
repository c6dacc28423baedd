// Tensor-map (TMA descriptor) helpers shared by the kernels that stage tiles with cp.async.bulk.tensor.
#pragma once
#include <cuda.h>   // CUtensorMap + the cuTensorMapEncodeTiled prototype (resolved at run time, no link dependency)
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace kt {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// driver entry point through the runtime: libkantts has no link-time libcuda dependency
inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) f = nullptr;
    return reinterpret_cast<EncodeTiledFn>(f);
  }();
  return fn;
}

// Tiled tensor map of a `rank`-D tensor (rank <= 5): dims and box innermost first, `strides` = byte strides of dims
// 1 .. rank - 1, unit element strides, no interleave; elements outside the tensor arrive as zeros.  `what` prefixes the
// error message.
inline int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, int rank, const void* base, const cuuint64_t* dims,
                             const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle,
                             CUtensorMapL2promotion l2, const char* what) {
  const EncodeTiledFn fn = encode_tiled_fn();
  KT_REQUIRE(fn != nullptr, "%s: the driver provides no cuTensorMapEncodeTiled", what);
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult r = fn(map, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  KT_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled failed (%d)", what, (int)r);
  return KT_OK;
}

// Split-bf16 planes of a [batch][t][nsub][c] fp32 tensor (split_planes, tc_common.cuh): [hi | lo][batch][t][nsub][c] bf16
// (single-pass bf16: the hi plane only).  plane_floats: workspace floats that `planes` planes occupy (half a float per element
// per plane), rounded up to 256 bytes.
inline long long plane_floats(long long batch, long long t, long long nsub, long long c, int planes = 2) {
  return ((batch * t * nsub * c * planes + 1) / 2 + 63) & ~63LL;
}

// Tensor map of residue class rho of such planes, time steps rho, rho + step, ...: 5-D boxes of box_c channels x nsub x box_t
// of those steps, SWIZZLE_128B; coordinates (channel, sub-sequence, step of the class, batch, plane), `nplanes` planes
inline int encode_plane_map(CUtensorMap* map, const __nv_bfloat16* planes, int batch, int t, int nsub, int c, int step, int rho,
                            int box_c, int box_t, const char* what, int nplanes = 2) {
  const long long n = (long long)batch * t * nsub * c;
  const cuuint64_t dims[5] = {(cuuint64_t)c, (cuuint64_t)nsub, (cuuint64_t)ceil_div(t - rho, step), (cuuint64_t)batch,
                              (cuuint64_t)nplanes};
  const cuuint64_t strides[4] = {(cuuint64_t)c * 2, (cuuint64_t)step * nsub * c * 2, (cuuint64_t)t * nsub * c * 2, (cuuint64_t)n * 2};
  const cuuint32_t box[5] = {(cuuint32_t)box_c, (cuuint32_t)nsub, (cuuint32_t)box_t, 1, 1};
  return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, planes + (long long)rho * nsub * c, dims, strides, box,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, what);
}

namespace tc {

// one 5-D box global -> shared (SASS UTMALDG.5D), completion (box bytes) on an mbarrier; out-of-range elements arrive as zeros
__device__ __forceinline__ void tma_load_5d(void* dst_smem, const CUtensorMap* map, int c0, int c1, int c2, int c3, int c4, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(
          (uint32_t)__cvta_generic_to_shared(dst_smem)),
      "l"(map), "r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// one 3-D box global -> shared
__device__ __forceinline__ void tma_load_3d(void* dst_smem, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                   (uint32_t)__cvta_generic_to_shared(dst_smem)),
               "l"(map), "r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

}  // namespace tc
}  // namespace kt
