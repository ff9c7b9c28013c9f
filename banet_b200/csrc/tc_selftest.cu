// Diagnostic: one 64-pixel k-tile through the exact TMA / tf32-MMA building blocks of the tensor-core build path.
//   D[128 x 160] = A^T R   with A [64 x 128] (TMA, 128B swizzle, as the basis tile lands) and
//   R [64 x 160] (written by SIMT stores into the same swizzled layout); fragments by load_a_frag / mma_step (tc_utils.cuh).
// mode 0: one tf32 pass (A truncated).  mode 1: plus a second pass with A_lo = A - trunc(A).
#include "common.cuh"
#include "tc_utils.cuh"
#include "tmap.h"

namespace banet {
using namespace tc;

constexpr int ST_PX = 64, ST_M = 128, ST_N = 160;

// 8 warps: warp w computes rows 16w .. 16w+15 of D, all 20 n8 column blocks
__global__ void __launch_bounds__(256, 1)
tc_selftest_kernel(const __grid_constant__ CUtensorMap tmapA, const float* __restrict__ Rg, float* __restrict__ Dg, int mode, int use_rna, int repeat)
{
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* sA = base;                       // 4 blocks x [64][128 B]   = 32 KB
    unsigned char* sAlo = base + 32768;             // same layout
    unsigned char* sR = base + 65536;               // 5 blocks x [64][128 B]   = 40 KB
    __shared__ __align__(8) uint64_t bar_full;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    if (tid == 0) { mbar_init(&bar_full, 1); fence_barrier_init(); }
    __syncthreads();

    if (tid == 0) {
        mbar_arrive_expect_tx(&bar_full, 32768);
        for (int blk = 0; blk < 4; ++blk) tma_load_2d(sA + blk * 8192, &tmapA, blk * 32, 0, &bar_full);
    }
    // R -> swizzled smem (float4 per 16-B chunk)
    for (int i = tid; i < ST_PX * (ST_N / 4); i += blockDim.x) {
        const int r = i / (ST_N / 4), c = i - r * (ST_N / 4);          // chunk c of row r
        float4 v = *reinterpret_cast<const float4*>(Rg + (size_t)r * ST_N + 4 * c);
        if (use_rna) { v.x = tf32_rna(v.x); v.y = tf32_rna(v.y); v.z = tf32_rna(v.z); v.w = tf32_rna(v.w); }
        *reinterpret_cast<float4*>(sR + (c >> 3) * 8192 + sw128_off(r, c & 7)) = v;
    }
    mbar_wait(&bar_full, 0);
    if (mode == 1) {
        for (int i = tid; i < ST_PX * 32; i += blockDim.x) {
            const int r = i >> 5, c = i & 31;
            const uint32_t off = (c >> 3) * 8192 + sw128_off(r, c & 7);
            float4 v = *reinterpret_cast<const float4*>(sA + off);
            v.x -= tf32_trunc(v.x); v.y -= tf32_trunc(v.y); v.z -= tf32_trunc(v.z); v.w -= tf32_trunc(v.w);
            *reinterpret_cast<float4*>(sAlo + off) = v;
        }
    }
    __syncthreads();

    constexpr int NQ = ST_N / 8;
    float acc[NQ][4];
#pragma unroll
    for (int q = 0; q < NQ; ++q) acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.f;
    for (int rep = 0; rep < repeat; ++rep)
        for (int pass = 0; pass <= mode; ++pass) {
            const uint32_t a = smem_u32(pass ? sAlo : sA), r = smem_u32(sR);
            for (int kk = 0; kk < ST_PX / 8; ++kk) {
                uint32_t af[4];
                load_a_frag(af, a, 16 * warp, kk, lane);
#pragma unroll
                for (int q = 0; q < NQ; ++q) mma_step(acc[q], af, r, 8 * q, kk, lane);
            }
        }
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int q = 0; q < NQ; ++q)
#pragma unroll
        for (int e = 0; e < 4; ++e) Dg[(size_t)(16 * warp + g + (e >> 1) * 8) * ST_N + 8 * q + 2 * t + (e & 1)] = acc[q][e];
}

}  // namespace banet

using namespace banet;

extern "C" int banet_tc_selftest(const float* A, const float* R, float* D, int mode, int use_rna, int repeat, banet_stream_t stream)
{
    BANET_REQUIRE(A && R && D, BANET_ERR_BAD_ARG, "tc_selftest: null pointer");
    CUtensorMap tm;
    int rc = make_tmap_basis_2d(&tm, A, false, ST_PX, ST_M, ST_PX, 32);
    if (rc) return rc;
    const size_t smem = 65536 + 40960 + 1024;
    cudaError_t e = cudaFuncSetAttribute(tc_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("tc_selftest smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    tc_selftest_kernel<<<1, 256, smem, (cudaStream_t)stream>>>(tm, R, D, mode, use_rna, repeat < 1 ? 1 : repeat);
    BANET_CUDA_LAUNCH_CHECK("tc_selftest_kernel launch");
    return BANET_OK;
}
