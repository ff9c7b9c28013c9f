// Host-side creation of TMA tensor maps through the driver entry point (no link-time libcuda dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include "common.cuh"

namespace banet {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_tiled()
{
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) {
        cudaGetLastError();
        return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeTiled>(p);
    return fn;
}

// Basis matrix [rows, cols] row-major (cols contiguous), fp32 or bf16; box = box_cols x box_rows.  fp32: 128B swizzle (16-byte chunk
// index XOR row & 7, tc_utils.cuh: sw128_off), box_cols*4 must be 128.  bf16: 64B swizzle (chunk index XOR (row >> 1) & 3, sw64_off),
// box_cols*2 must be 64.
inline int make_tmap_basis_2d(CUtensorMap* out, const void* base, bool bf16, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols)
{
    PFN_encodeTiled enc = get_encode_tiled();
    BANET_REQUIRE(enc, BANET_ERR_CUDA, "cuTensorMapEncodeTiled driver entry point not available");
    const uint64_t es = bf16 ? 2 : 4;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstr[1] = {cols * es};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, bf16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    BANET_REQUIRE(r == CUDA_SUCCESS, BANET_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu", (int)r,
                  (unsigned long long)rows, (unsigned long long)cols);
    return BANET_OK;
}

// Basis tensor [planes, rows, cols] (cols contiguous, dense), fp32 or bf16: box = box_cols x box_rows x box_planes, same swizzles.
// Used for the basis of a dense pixel grid: cols = K, rows = grid_w (x), planes = nb*grid_h (y); an 8x8 pixel tile is one box.
inline int make_tmap_basis_3d(CUtensorMap* out, const void* base, bool bf16, uint64_t planes, uint64_t rows, uint64_t cols,
                              uint32_t box_planes, uint32_t box_rows, uint32_t box_cols)
{
    PFN_encodeTiled enc = get_encode_tiled();
    BANET_REQUIRE(enc, BANET_ERR_CUDA, "cuTensorMapEncodeTiled driver entry point not available");
    const uint64_t es = bf16 ? 2 : 4;
    cuuint64_t gdim[3] = {cols, rows, planes};
    cuuint64_t gstr[2] = {cols * es, rows * cols * es};
    cuuint32_t box[3] = {box_cols, box_rows, box_planes};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(out, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, bf16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    BANET_REQUIRE(r == CUDA_SUCCESS, BANET_ERR_CUDA, "cuTensorMapEncodeTiled(3d) failed (%d)", (int)r);
    return BANET_OK;
}

}  // namespace banet
