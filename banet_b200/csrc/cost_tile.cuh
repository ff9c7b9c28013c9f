// The 64-point tile of the feature-metric cost kernels: lm_cost_kernel / lm_cost_bwd_kernel (lm_cost.cu, one pair per tile) and
// keyframe_cost_kernel / keyframe_cost_bwd_kernel (lm_window_cost.cu, one keyframe tile walked over its window's frames): the per-point
// records of a tile, and the value-only residual norm of one point (S2) and the tile's fp64 sum (S3) in lm_cost_kernel's statements and
// order, so both layouts give the same bits.  lm_cost_kernel keeps its own copy of S2 and S3 inline: calling these two changes its register
// allocation (cuobjdump -sass), and its machine code stays as it was.
#pragma once
#include "common.cuh"
#include "point.cuh"

namespace banet {

constexpr int COST_TILE = 64;
constexpr int COST_THREADS = 256;
constexpr int COST_WARPS = COST_THREADS / 32;
// records [CR_ARRAYS][COST_TILE]: point index (or -1), tap corner, fractions, mask, depth, pixel gradient, the point's cost term
enum { CR_IDX = 0, CR_X0, CR_Y0, CR_DX, CR_DY, CR_MASK, CR_DT, CR_DU, CR_DV, CR_VAL, CR_ARRAYS };

__device__ __forceinline__ Taps cost_taps(const float* rec, int i, int h, int w) {
    return Taps(__float_as_int(rec[CR_X0 * COST_TILE + i]), __float_as_int(rec[CR_Y0 * COST_TILE + i]), rec[CR_DX * COST_TILE + i],
                rec[CR_DY * COST_TILE + i], h, w);
}

// S2 of the in-bounds point of record i, lanes over channels: s = sum_c d_c^2 against the pair's map img (c2 channels per texel, the first C
// read), conv1's row c1; four channels per lane when vec4, else one.  Returned summed over the warp.
template <typename TF>
__device__ __forceinline__ float cost_point_s(const TF* img, const TF* c1, const float* rec, int i, int h, int w, int c2, int C, int vec4, int lane)
{
    const ValueTaps vt(cost_taps(rec, i, h, w), w, c2);
    float s = 0.f;
    if (vec4) {
        for (int c = lane * 4; c < C; c += 32 * 4) { ChanVec<4, TF> f1; f1.load_stream(c1 + c); vt.squares<4>(img, f1, c, s); }
    } else {
        for (int c = lane; c < C; c += 32) { ChanVec<1, TF> f1; f1.load_stream(c1 + c); vt.squares<1>(img, f1, c, s); }
    }
    return warp_sum(s);
}

// S3, warp 0: the tile's 64 cost terms and in-bounds count in fp64, in a fixed order (lane pairs i, i + 32, then a butterfly), into its
// slot (one writer)
__device__ __forceinline__ void cost_tile_sum(const float* rec, int lane, double* slot)
{
    double v = (double)rec[CR_VAL * COST_TILE + lane] + (double)rec[CR_VAL * COST_TILE + lane + 32];
    double n = (double)rec[CR_MASK * COST_TILE + lane] + (double)rec[CR_MASK * COST_TILE + lane + 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { v += __shfl_xor_sync(0xffffffffu, v, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
    if (lane == 0) { slot[0] = v; slot[1] = n; }
}

}  // namespace banet
