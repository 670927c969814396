// Shared by the kernels that run a 3x3 conv straight out of a TMA halo (heads.cu: the output heads, dcnv2_tc.cu: the
// offset/mask conv of the DCN block kernel): the 4-D tensor-map halo load and the driver's tensor-map encoder.
//
// A halo is loaded as 8-channel slabs [y][x][8 ch] of a bf16 channels-last [B][H][W][C] tensor; the out-of-bounds
// fill of the tensor map is the conv's zero padding.  The 8 pixels of a wgmma core-matrix row group are 8 consecutive
// halo pixels of one row, so the A operand of tap (dy, dx) is the slab itself read through a descriptor shifted by
// (dy * halo_width + dx) * 16 bytes: no im2col tile is built.
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_bf16.h>

#include "dcnv2_tc.cuh"

namespace cnb {

// One box of a 4-D tensor map (channel, x, y, image) into shared memory (128-byte aligned), completing on `bar`
__device__ __forceinline__ void tma_load_4d(void *dst, const CUtensorMap *map, int c0, int c1, int c2, int c3,
                                            uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
      "r"(smem_u32(bar))
      : "memory");
}

// cuTensorMapEncodeTiled from the driver (no libcuda link); nullptr when the driver does not have it
inline PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      (void)cudaGetLastError();
      p = nullptr;
    }
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }();
  return fn;
}

// Tensor map of a bf16 channels-last [b][h][w][c] tensor whose box is one 8-channel slab of a box_x x box_y halo;
// out-of-bounds elements read as zero.  Returns the driver's result (CUDA_ERROR_NOT_SUPPORTED without an encoder).
inline CUresult encode_halo_map(CUtensorMap *map, const void *x, int b, int c, int h, int w, int box_x, int box_y) {
  PFN_cuTensorMapEncodeTiled_v12000 encode = tensor_map_encoder();
  if (encode == nullptr) return CUDA_ERROR_NOT_SUPPORTED;
  cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)b};
  cuuint64_t strides[3] = {(cuuint64_t)c * 2, (cuuint64_t)w * c * 2, (cuuint64_t)h * w * c * 2};
  cuuint32_t box[4] = {8, (cuuint32_t)box_x, (cuuint32_t)box_y, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  return encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(x), dims, strides, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

}  // namespace cnb
