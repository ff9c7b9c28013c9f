// mma_role.cuh — the MMA warpgroup of the tensor-core build kernel (generation 6): D = A^T R of every tile by mma.sync
// m16n8k8 tf32, each 8-pixel product added round-to-nearest into register accumulators that live for the whole pair span, one slot
// write per span.
//
// Work split (lm_reduce reads the lower block triangle of H_dd only and mirrors it): m-block mb (16 rows of D) needs the columns
// 0 .. 16mb+15 plus the [v | t] block (columns KR .. KR+7).  At K = 128 warp mw takes m-blocks mw and 7-mw; at K = 64 / 32 one
// m-block per warp (none for warps >= K / 16).  The split is a template argument: every fragment address is a lane offset plus an
// immediate, and the contraction of a tile is straight-line code without branches.
//
// Fragment <-> column mapping (tests/test_mma_fragment_layout.py checks it).  The order of the rows and columns inside an accumulator block
// is free, because the span write below places every element by its (row, column); the pixel order inside an 8-pixel step is kept.
//   A, m-block mb: fragment rows g and g+8 are basis columns 16mb+2g and 16mb+2g+1, so (a0, a1) at pixel t and (a2, a3) at pixel
//     t+4 are one LDS.64 each.  (An m-block's 16 columns are 4 chunks of one half of the 128-B row, and rows 0..3 of the swizzle
//     permute chunks inside a half: these loads keep the 2-way bank conflict of any fragment walk over one m-block.)
//   R, full column group G (columns 32G .. 32G+31, one swizzle block): four accumulator blocks j = 0..3; fragment column g of block j
//     is column 32G + 4c(g) + j with c(g) = (g >> 1) | ((g & 1) << 2).  Lane (g, t) reads 16-B chunk c(g) of pixel rows t and t+4:
//     one LDS.128 each gives b0 / b1 of all four blocks.  Quarter-warp q holds g = 2q, 2q+1, i.e. chunks q and q+4 XOR t < 4: 8
//     distinct bank groups, conflict-free.
//   R, half group (columns 32G .. 32G+15, G = mb / 2, the last columns of an m-block with mb even): two accumulator blocks j = 0, 1;
//     fragment column g of block j is column 32G + 2g + j, one LDS.64 per pixel row (the walk of the A pairs, same 2-way conflict).
//   [v | t] block: fragment column g is column KR + g, as the algebra warps write it; scalar loads.
//   A on a bf16 basis (BB; 64-B rows, 64B swizzle): columns 2g and 2g+1 are one 32-bit word, so (a0, a1) at pixel t and (a2, a3) at
//     pixel t+4 are one LDS.32 each, widened by a shift and a mask (exact tf32 values).  Rows t and t+2 are 128 B apart: the same 2-way
//     bank conflict.  The split-A pass is skipped (A_lo = 0); the passes left keep their order.
// Accumulator element e (fragment row g + 8(e >> 1), column 2t + (e & 1)) holds row i = 16mb + 2g + (e >> 1) and column
//   n = 32G + 4t + 16(e & 1) + j (full group), 32G + 4t + 2(e & 1) + j (half group), KR + 2t + (e & 1) ([v | t]).
#pragma once
#include "common.cuh"
#include "lm_build.h"
#include "tc_utils.cuh"

namespace banet { namespace tc {

// d = A x B from zero (the tensor core's product of one 8-pixel step); no side effects, so the compiler may schedule it freely
__device__ __forceinline__ void mma_tf32_m16n8k8_z(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(0.f));
}
// acc += (8-pixel product), added in fp32 round-to-nearest: the tensor core's own fp32 accumulation truncates (biased toward zero,
// see tests/test_gpu_tensorcore.py), which over the thousands of steps of a pair span would bias H_dd
__device__ __forceinline__ void mma_add_rn(float (&acc)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    float p[4];
    mma_tf32_m16n8k8_z(p, a, b0, b1);
    acc[0] += p[0]; acc[1] += p[1]; acc[2] += p[2]; acc[3] += p[3];
}
__device__ __forceinline__ uint32_t tf32_bits(float x) { return __float_as_uint(x) & 0xFFFFE000u; }

// full column groups of m-block mb (-1: no m-block), and whether it ends on a half group
__host__ __device__ constexpr int mma_full_groups(int mb) { return mb < 0 ? 0 : (mb + 1) / 2; }
__host__ __device__ constexpr bool mma_half_group(int mb) { return mb >= 0 && (mb & 1) == 0; }

template <int MB> struct MmaAcc {                      // accumulators of one m-block: full groups, half group, [v | t] block
    static constexpr int NF = mma_full_groups(MB);
    static constexpr bool HALF = mma_half_group(MB);
    float h[NF > 0 ? NF : 1][4][4];
    float hh[2][4];
    float x[4];
    __device__ __forceinline__ void zero() {
#pragma unroll
        for (int G = 0; G < NF; ++G)
#pragma unroll
            for (int j = 0; j < 4; ++j) h[G][j][0] = h[G][j][1] = h[G][j][2] = h[G][j][3] = 0.f;
        hh[0][0] = hh[0][1] = hh[0][2] = hh[0][3] = hh[1][0] = hh[1][1] = hh[1][2] = hh[1][3] = 0.f;
        x[0] = x[1] = x[2] = x[3] = 0.f;
    }
    // slot of the span: H_dd column-major (hdd_transposed), ext rows [v | t]
    template <int KR> __device__ __forceinline__ void write(float* slot, int g, int t) {
        if constexpr (MB >= 0) {
            const int i0 = 16 * MB + 2 * g;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int i = i0 + (e >> 1);
#pragma unroll
                for (int G = 0; G < NF; ++G)
#pragma unroll
                    for (int j = 0; j < 4; ++j) slot[(size_t)(32 * G + 16 * (e & 1) + 4 * t + j) * KR + i] = h[G][j][e];
                if constexpr (HALF) {
#pragma unroll
                    for (int j = 0; j < 2; ++j) slot[(size_t)(32 * NF + 2 * (e & 1) + 4 * t + j) * KR + i] = hh[j][e];
                }
                const int n = 2 * t + (e & 1);
                if (n < 7) slot[KR * KR + n * KR + i] = x[e];
            }
        }
        zero();
    }
};

template <class SM, int STAGE_A, int MODE, int KR, int MB0, int MB1, bool BB>
__device__ __forceinline__ void mma_warp(const BuildParams& prm, const unsigned char* base, uint64_t* fullB, uint64_t* rready,
                                         uint64_t* rfree, long long t_begin, int ntiles, int lane)
{
    constexpr int NST = SM::NST, EXTB = KR / 32;
    constexpr int NG0 = mma_full_groups(MB0), NG1 = mma_full_groups(MB1), NG = NG0 > NG1 ? NG0 : NG1;
    constexpr bool H0 = mma_half_group(MB0), H1 = mma_half_group(MB1);
    const int g = lane >> 2, t = lane & 3;
    // lane byte offsets at pixel row t of an 8-pixel step (row t+4: +512, and bit 2 of the 16-B chunk flips)
    const uint32_t oa = t * 128 + (((g >> 1) ^ t) << 4) + (g & 1) * 8;                 // A: columns 2g, 2g+1 of a low-half m-block
    const uint32_t ob0 = t * 128 + ((((g >> 1) | ((g & 1) << 2)) ^ t) << 4);          // R: chunk c(g)
    const uint32_t ob1 = (ob0 ^ 64) + 512;
    const uint32_t ox = EXTB * 8192 + t * 128 + (((g >> 2) ^ t) << 4) + (g & 3) * 4;    // [v | t]: column KR + g
    const uint32_t oab = t * 64 + (((g >> 2) ^ (t >> 1)) << 4) + (g & 3) * 4;           // bf16 A: columns 2g, 2g+1 of a low-half m-block
    MmaAcc<MB0> acc0;
    MmaAcc<MB1> acc1;
    acc0.zero(); acc1.zero();
    int span = 0;
    int rr = (ntiles > 0) ? (int)((unsigned)t_begin % (unsigned)prm.tiles_per_pair) : 0;
    for (int j = 0; j < ntiles; ++j) {
        const int s = j % NST;
        mbar_wait_parked(rready, j & 1);
        mbar_wait_parked(&fullB[s], (j / NST) & 1);      // orders the TMA writes of the stage before the fragment loads
        const unsigned char* ahi = base + SM::off_A + s * STAGE_A;
#pragma unroll 1
        for (int pass = 0; pass < MODE; ++pass) {        // hi x hi, then A_lo x R, then A x R_lo, into the same accumulators
            if constexpr (BB) { if (pass == 1) continue; }
            const unsigned char* a = pass == 1 ? base + SM::off_Alo : ahi;
            const unsigned char* r = base + (pass == 2 ? SM::off_Rlo : SM::off_R);
#pragma unroll 1
            for (int kk = 0; kk < 8; ++kk) {
                const unsigned char* ak = a + kk * (BB ? 512 : 1024);
                const unsigned char* rk = BB ? r + kk * 1024 : ak + (r - a);
                uint32_t f0[4], f1[4];
                if constexpr (BB) {
                    if constexpr (MB0 >= 0) {
                        const uint32_t lo = *reinterpret_cast<const uint32_t*>(ak + (MB0 >> 1) * 4096 + oab + 32 * (MB0 & 1));
                        const uint32_t hi = *reinterpret_cast<const uint32_t*>(ak + (MB0 >> 1) * 4096 + 256 + oab + 32 * ((MB0 & 1) ^ 1));
                        f0[0] = lo << 16; f0[1] = lo & 0xFFFF0000u; f0[2] = hi << 16; f0[3] = hi & 0xFFFF0000u;
                    }
                    if constexpr (MB1 >= 0) {
                        const uint32_t lo = *reinterpret_cast<const uint32_t*>(ak + (MB1 >> 1) * 4096 + oab + 32 * (MB1 & 1));
                        const uint32_t hi = *reinterpret_cast<const uint32_t*>(ak + (MB1 >> 1) * 4096 + 256 + oab + 32 * ((MB1 & 1) ^ 1));
                        f1[0] = lo << 16; f1[1] = lo & 0xFFFF0000u; f1[2] = hi << 16; f1[3] = hi & 0xFFFF0000u;
                    }
                } else {
                if constexpr (MB0 >= 0) {
                    const uint2 lo = *reinterpret_cast<const uint2*>(ak + (MB0 >> 1) * 8192 + oa + 64 * (MB0 & 1));
                    const uint2 hi = *reinterpret_cast<const uint2*>(ak + (MB0 >> 1) * 8192 + 512 + oa + 64 * ((MB0 & 1) ^ 1));
                    f0[0] = lo.x & 0xFFFFE000u; f0[1] = lo.y & 0xFFFFE000u; f0[2] = hi.x & 0xFFFFE000u; f0[3] = hi.y & 0xFFFFE000u;
                }
                if constexpr (MB1 >= 0) {
                    const uint2 lo = *reinterpret_cast<const uint2*>(ak + (MB1 >> 1) * 8192 + oa + 64 * (MB1 & 1));
                    const uint2 hi = *reinterpret_cast<const uint2*>(ak + (MB1 >> 1) * 8192 + 512 + oa + 64 * ((MB1 & 1) ^ 1));
                    f1[0] = lo.x & 0xFFFFE000u; f1[1] = lo.y & 0xFFFFE000u; f1[2] = hi.x & 0xFFFFE000u; f1[3] = hi.y & 0xFFFFE000u;
                }
                }
#pragma unroll
                for (int G = 0; G < NG; ++G) {
                    const float4 v0 = *reinterpret_cast<const float4*>(rk + G * 8192 + ob0);
                    const float4 v1 = *reinterpret_cast<const float4*>(rk + G * 8192 + ob1);
                    const uint32_t b0[4] = {tf32_bits(v0.x), tf32_bits(v0.y), tf32_bits(v0.z), tf32_bits(v0.w)};
                    const uint32_t b1[4] = {tf32_bits(v1.x), tf32_bits(v1.y), tf32_bits(v1.z), tf32_bits(v1.w)};
#pragma unroll
                    for (int jb = 0; jb < 4; ++jb) {
                        if (G < NG0) mma_add_rn(acc0.h[G][jb], f0, b0[jb], b1[jb]);
                        if (G < NG1) mma_add_rn(acc1.h[G][jb], f1, b0[jb], b1[jb]);
                    }
                }
                if constexpr (H0 || H1) {                    // at most one m-block of a warp is even
                    constexpr int GH = H0 ? NG0 : NG1;
                    const uint2 v0 = *reinterpret_cast<const uint2*>(rk + GH * 8192 + oa);
                    const uint2 v1 = *reinterpret_cast<const uint2*>(rk + GH * 8192 + 512 + oa + 64);
                    const uint32_t b0[2] = {v0.x & 0xFFFFE000u, v0.y & 0xFFFFE000u}, b1[2] = {v1.x & 0xFFFFE000u, v1.y & 0xFFFFE000u};
#pragma unroll
                    for (int jb = 0; jb < 2; ++jb) {
                        if constexpr (H0) mma_add_rn(acc0.hh[jb], f0, b0[jb], b1[jb]);
                        else mma_add_rn(acc1.hh[jb], f1, b0[jb], b1[jb]);
                    }
                }
                if constexpr (MB0 >= 0) {
                    const uint32_t x0 = tf32_bits(*reinterpret_cast<const float*>(rk + ox));
                    const uint32_t x1 = tf32_bits(*reinterpret_cast<const float*>(rk + ox + 576));
                    mma_add_rn(acc0.x, f0, x0, x1);
                    if constexpr (MB1 >= 0) mma_add_rn(acc1.x, f1, x0, x1);
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(rfree);
        const bool last_of_pair = (++rr == prm.tiles_per_pair) || (j == ntiles - 1);
        if (rr == prm.tiles_per_pair) rr = 0;
        if (last_of_pair) {
            float* slot = prm.partials + ((size_t)blockIdx.x * prm.max_span + span) * prm.slot_floats;
            acc0.template write<KR>(slot, g, t);
            acc1.template write<KR>(slot, g, t);
            ++span;
        }
    }
}

// The MMA warpgroup: dispatch once on the warp index mw (0..3) into its compile-time work split.
template <class SM, int STAGE_A, int MODE, int KR, bool BB = false>
__device__ __forceinline__ void mma_role(const BuildParams& prm, const unsigned char* base, uint64_t* fullB, uint64_t* rready,
                                         uint64_t* rfree, long long t_begin, int ntiles, int mw, int lane)
{
    constexpr int NMB = KR / 16;
#define BANET_MMA_WARP(A, B) mma_warp<SM, STAGE_A, MODE, KR, A, B, BB>(prm, base, fullB, rready, rfree, t_begin, ntiles, lane)
    if constexpr (NMB == 8) {
        switch (mw) { case 0: BANET_MMA_WARP(0, 7); break; case 1: BANET_MMA_WARP(1, 6); break;
                      case 2: BANET_MMA_WARP(2, 5); break; default: BANET_MMA_WARP(3, 4); break; }
    } else if constexpr (NMB == 4) {
        switch (mw) { case 0: BANET_MMA_WARP(0, -1); break; case 1: BANET_MMA_WARP(1, -1); break;
                      case 2: BANET_MMA_WARP(2, -1); break; default: BANET_MMA_WARP(3, -1); break; }
    } else {
        static_assert(NMB == 2, "K = 128, 64 or 32");
        switch (mw) { case 0: BANET_MMA_WARP(0, -1); break; case 1: BANET_MMA_WARP(1, -1); break; default: BANET_MMA_WARP(-1, -1); break; }
    }
#undef BANET_MMA_WARP
}

}}  // namespace banet::tc
