// Feature-metric cost of a level and its backward (include/banet_abi.h, banet_lm_cost / banet_lm_cost_bwd).
//
//   s_n = sum_c d_{n,c}^2,  d = conv1 - F2(pi(p, D + B.W; R, T)),   cost[b] = sum_n c_n rho(s_n) over the in-bounds points of pair b
//
// with the build's warp, mask and bilinear sample of the F2 values (point.cuh), c_n the point weight and rho the level's robust loss
// (common.cuh: rho(s) = s without one).  Nothing per point is kept between the kernels but the optional s and mask outputs.
//
// lm_cost_kernel: persistent over tiles of 64 points (linear, or 8 x 8 raster tiles with a grid hint), four stages per tile:
//   S0 stage the tile's basis rows (coalesced, widened), S1 thread per point: D + b.W (basis_dot, the build's arithmetic: nvalid is the
//   build's), projection, mask and taps, S2 warp per point: the value taps of every channel, s by a warp sum, c rho(s), S3 one warp sums
//   the tile's 64 values in fp64 in a fixed order and writes the tile's slot (one writer).  lm_cost_reduce_kernel sums a pair's slots in
//   fp64 in a fixed order, so the cost does not depend on the grid or on what the workspace held.
// lm_cost_bwd_kernel: the same S0 / S1, then warp per point: s again (ROBUST only: rho' needs it before the channel pass), and one
//   channel pass that stores dconv1 = dd = 2 dcost c rho'(s) d (one writer), scatters -w_tau dd into the four value taps of dconv2
//   (atomics) and accumulates the pixel gradient from the tap differences; thread per point: the geometry backward (GeomGrad with dJ = 0)
//   -> dD, and dR, dT in per-thread sums; dB = dDt W (one writer) and dW = sum_n dDt b in per-column sums, committed at a pair change.
#include "common.cuh"
#include "features.cuh"
#include "lm_build.h"
#include "point.cuh"
#include "cost_tile.cuh"
#include <string.h>

namespace banet {

struct CostParams {
    int nb, N, C, K, KP, h, w;
    const void *conv1, *conv2;                   // element type: the kernel's TF
    const float *intr, *p, *D;
    const void* B;                               // element type: the kernel's TB
    const float *R, *T, *W, *weight;
    int robust;
    float robust_scale;
    int grid_w, grid_h, tiles_x, tiles_per_pair, vec4;
    long long total_tiles;
    double* partials;                            // forward: [total_tiles][2] = (sum c rho(s), in-bounds count) per tile
    float *s_out, *mask_out;                     // forward, optional
    const float* dcost;                          // backward
    float *dconv1, *dconv2, *dD, *dB, *dR, *dT, *dW, *dweight;
};

// smem (floats): Bs [64][KP+4] | W [KP] | pose [16] | records [CR_ARRAYS][64]
static size_t cost_smem_bytes(int KP) { return (size_t)((KP > 0 ? COST_TILE * (KP + 4) + KP : 0) + 16 + CR_ARRAYS * COST_TILE) * sizeof(float); }

// point i of tile r of a pair, or -1: 64 consecutive points, or the 8 x 8 raster tile (r % tiles_x, r / tiles_x) of the grid hint
__device__ __forceinline__ int cost_point(const CostParams& prm, int r, int i) {
    if (prm.grid_w > 0) {
        const int gx = (r % prm.tiles_x) * 8 + (i & 7), gy = (r / prm.tiles_x) * 8 + (i >> 3);
        return (gx < prm.grid_w && gy < prm.grid_h) ? gy * prm.grid_w + gx : -1;
    }
    const int n = r * COST_TILE + i;
    return n < prm.N ? n : -1;
}

// S0 and S1 of both kernels: stage tile r of pair b and derive each point's depth, mask and taps into the records (thread per point)
template <typename TB>
__device__ __forceinline__ void cost_tile_geometry(const CostParams& prm, int b, int r, float* Bs, const float* sW, const float* sPose, float* rec)
{
    const int tid = threadIdx.x, K = prm.K, KP = prm.KP, LDB = KP + 4, N = prm.N;
    if (tid < COST_TILE) rec[CR_IDX * COST_TILE + tid] = __int_as_float(cost_point(prm, r, tid));
    __syncthreads();
    if (KP > 0) {
        const TB* Bg = static_cast<const TB*>(prm.B) + (size_t)b * N * K;
        if ((K & 3) == 0 && (sizeof(TB) == 4 || (reinterpret_cast<uintptr_t>(prm.B) & 7) == 0)) {
            const int k4 = K >> 2, kp4 = KP >> 2;
            for (int i = tid; i < COST_TILE * kp4; i += COST_THREADS) {
                const int n = i / kp4, q = i - n * kp4, pt = __float_as_int(rec[CR_IDX * COST_TILE + n]);
                ChanVec<4, TB> v;
                if (pt >= 0 && q < k4) v.load_stream(Bg + (size_t)pt * K + 4 * q);
                else v.v[0] = v.v[1] = v.v[2] = v.v[3] = 0.f;
                *reinterpret_cast<float4*>(Bs + n * LDB + 4 * q) = make_float4(v.v[0], v.v[1], v.v[2], v.v[3]);
            }
        } else {
            for (int i = tid; i < COST_TILE * KP; i += COST_THREADS) {
                const int n = i / KP, k = i - n * KP, pt = __float_as_int(rec[CR_IDX * COST_TILE + n]);
                Bs[n * LDB + k] = (pt >= 0 && k < K) ? ld_stream_elem(Bg + (size_t)pt * K + k) : 0.f;
            }
        }
    }
    __syncthreads();
    if (tid < COST_TILE) {
        const int pt = __float_as_int(rec[CR_IDX * COST_TILE + tid]);
        float mask = 0.f, dx = 0.f, dy = 0.f, Dt = 0.f;
        int x0 = 0, y0 = 0;
        if (pt >= 0) {
            const float* pp = prm.p + (size_t)b * 3 * N + pt;
            Dt = prm.D[(size_t)b * N + pt];
            if (KP > 0) Dt += basis_dot_padded(Bs + tid * LDB, sW, KP);
            const Projection pr(sPose, pp[0], pp[N], pp[2 * (size_t)N], Dt);
            if (pr.in_bounds(prm.h, prm.w)) {
                mask = 1.f;
                tap_corner(pr.u, pr.v, x0, y0, dx, dy);
            }
        }
        rec[CR_X0 * COST_TILE + tid] = __int_as_float(x0); rec[CR_Y0 * COST_TILE + tid] = __int_as_float(y0);
        rec[CR_DX * COST_TILE + tid] = dx; rec[CR_DY * COST_TILE + tid] = dy; rec[CR_MASK * COST_TILE + tid] = mask; rec[CR_DT * COST_TILE + tid] = Dt;
    }
    __syncthreads();
}

// pose (R 9 | T 3 | intr 4) and W (padded to KP with zeros) of pair b
__device__ __forceinline__ void cost_pair_constants(const CostParams& prm, int b, float* sW, float* sPose)
{
    const int tid = threadIdx.x;
    if (tid < 9) sPose[tid] = prm.R[(size_t)b * 9 + tid];
    else if (tid < 12) sPose[tid] = prm.T[(size_t)b * 3 + tid - 9];
    else if (tid < 16) sPose[tid] = prm.intr[(size_t)b * 4 + tid - 12];
    for (int k = tid; k < prm.KP; k += COST_THREADS) sW[k] = (k < prm.K) ? prm.W[(size_t)b * prm.K + k] : 0.f;
}

// TF: feature element type; TB: basis element type; FLY: conv2 is F2 only (C channels per texel), else [F2|gx|gy] (3C, only the first C
// are read); ROBUST: the level has a robust loss (rho, rho'), else rho(s) = s
template <typename TF, typename TB, bool FLY, bool ROBUST>
__global__ void __launch_bounds__(COST_THREADS, 4)
lm_cost_kernel(const CostParams prm)
{
    extern __shared__ __align__(16) float smem[];
    const int KP = prm.KP;
    float* Bs = smem;
    float* sW = Bs + (KP > 0 ? COST_TILE * (KP + 4) : 0);
    float* sPose = sW + KP;
    float* rec = sPose + 16;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = prm.N, C = prm.C, h = prm.h, w = prm.w, c2 = FLY ? C : 3 * C;
    const long long t_begin = part_begin(prm.total_tiles, gridDim.x, blockIdx.x);
    const long long t_end = part_begin(prm.total_tiles, gridDim.x, blockIdx.x + 1);
    int cur_b = -1;
    for (long long t = t_begin; t < t_end; ++t) {
        const int b = (int)(t / prm.tiles_per_pair), r = (int)(t - (long long)b * prm.tiles_per_pair);
        if (b != cur_b) { cost_pair_constants(prm, b, sW, sPose); cur_b = b; }     // visible after the first barrier of the tile
        cost_tile_geometry<TB>(prm, b, r, Bs, sW, sPose, rec);
        // ---- S2: warp per point, lanes over channels -----------------------------------------------------------------------------------
        const TF* img = static_cast<const TF*>(prm.conv2) + (size_t)b * h * w * c2;
        for (int i = warp; i < COST_TILE; i += COST_WARPS) {
            const int pt = __float_as_int(rec[CR_IDX * COST_TILE + i]);
            if (pt < 0) { if (lane == 0) rec[CR_VAL * COST_TILE + i] = 0.f; continue; }
            const size_t gi = (size_t)b * N + pt;
            float val = 0.f, s = 0.f;
            if (rec[CR_MASK * COST_TILE + i] != 0.f) {
                const ValueTaps vt(cost_taps(rec, i, h, w), w, c2);
                const TF* c1 = static_cast<const TF*>(prm.conv1) + gi * C;
                if (prm.vec4) {
                    for (int c = lane * 4; c < C; c += 32 * 4) { ChanVec<4, TF> f1; f1.load_stream(c1 + c); vt.squares<4>(img, f1, c, s); }
                } else {
                    for (int c = lane; c < C; c += 32) { ChanVec<1, TF> f1; f1.load_stream(c1 + c); vt.squares<1>(img, f1, c, s); }
                }
                s = warp_sum(s);
                const float cn = prm.weight ? __ldg(prm.weight + gi) : 1.f;
                val = cn * (ROBUST ? robust_rho(prm.robust, prm.robust_scale, s) : s);
            }
            if (lane == 0) {
                rec[CR_VAL * COST_TILE + i] = val;
                if (prm.s_out) prm.s_out[gi] = s;
                if (prm.mask_out) prm.mask_out[gi] = rec[CR_MASK * COST_TILE + i];
            }
        }
        __syncthreads();
        // ---- S3: the tile's sum in fp64, fixed order (lane pairs i, i + 32, then a butterfly), one writer -------------------------------
        if (warp == 0) {
            double v = (double)rec[CR_VAL * COST_TILE + lane] + (double)rec[CR_VAL * COST_TILE + lane + 32];
            double n = (double)rec[CR_MASK * COST_TILE + lane] + (double)rec[CR_MASK * COST_TILE + lane + 32];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { v += __shfl_xor_sync(0xffffffffu, v, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
            if (lane == 0) { prm.partials[2 * t] = v; prm.partials[2 * t + 1] = n; }
        }
        // the next tile's first barrier orders these reads before its records are rewritten
    }
}

// warp per pair: lane l sums the pair's slots l, l + 32, ... in fp64, then a butterfly; the same order at every grid and batch size
__global__ void __launch_bounds__(256)
lm_cost_reduce_kernel(const double* __restrict__ partials, int nb, int tiles_per_pair, float* __restrict__ cost, float* __restrict__ nvalid)
{
    const int lane = threadIdx.x & 31;
    for (long long b = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < nb; b += ((long long)gridDim.x * blockDim.x) >> 5) {
        const double* sl = partials + (size_t)b * tiles_per_pair * 2;
        double v = 0.0, n = 0.0;
        for (int i = lane; i < tiles_per_pair; i += 32) { v += sl[2 * i]; n += sl[2 * i + 1]; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { v += __shfl_xor_sync(0xffffffffu, v, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
        if (lane == 0) { cost[b] = (float)v; nvalid[b] = (float)n; }
    }
}

template <typename TF, typename TB, bool FLY, bool ROBUST>
__global__ void __launch_bounds__(COST_THREADS, 2)
lm_cost_bwd_kernel(const CostParams prm)
{
    extern __shared__ __align__(16) float smem[];
    const int KP = prm.KP, K = prm.K, LDB = KP + 4;
    float* Bs = smem;
    float* sW = Bs + (KP > 0 ? COST_TILE * LDB : 0);
    float* sPose = sW + KP;
    float* rec = sPose + 16;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = prm.N, C = prm.C, h = prm.h, w = prm.w, c2 = FLY ? C : 3 * C;
    const long long t_begin = part_begin(prm.total_tiles, gridDim.x, blockIdx.x);
    const long long t_end = part_begin(prm.total_tiles, gridDim.x, blockIdx.x + 1);
    int cur_b = -1;
    float dc = 0.f;
    // pair-level sums: dR, dT by the point threads (tid < 64), dW column tid (tid < K); committed with atomics at a pair change
    float accR[9], accT[3], accW = 0.f;
#pragma unroll
    for (int i = 0; i < 9; ++i) accR[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) accT[i] = 0.f;
    auto commit = [&](int b) {
        if (tid < COST_TILE) {
#pragma unroll
            for (int i = 0; i < 9; ++i) { const float v = warp_sum(accR[i]); if (lane == 0) atomicAdd(prm.dR + (size_t)b * 9 + i, v); accR[i] = 0.f; }
#pragma unroll
            for (int i = 0; i < 3; ++i) { const float v = warp_sum(accT[i]); if (lane == 0) atomicAdd(prm.dT + (size_t)b * 3 + i, v); accT[i] = 0.f; }
        }
        if (tid < K) atomicAdd(prm.dW + (size_t)b * K + tid, accW);
        accW = 0.f;
    };

    for (long long t = t_begin; t < t_end; ++t) {
        const int b = (int)(t / prm.tiles_per_pair), r = (int)(t - (long long)b * prm.tiles_per_pair);
        if (b != cur_b) {
            if (cur_b >= 0) commit(cur_b);
            cost_pair_constants(prm, b, sW, sPose);
            dc = __ldg(prm.dcost + b);
            cur_b = b;
        }
        cost_tile_geometry<TB>(prm, b, r, Bs, sW, sPose, rec);
        // ---- warp per point, lanes over channels: dd, dconv1, the taps of dconv2, the pixel gradient -------------------------------------
        const TF* img = static_cast<const TF*>(prm.conv2) + (size_t)b * h * w * c2;
        float* dimg = prm.dconv2 + (size_t)b * h * w * c2;
        for (int i = warp; i < COST_TILE; i += COST_WARPS) {
            const int pt = __float_as_int(rec[CR_IDX * COST_TILE + i]);
            if (pt < 0) continue;
            const size_t gi = (size_t)b * N + pt;
            const TF* c1 = static_cast<const TF*>(prm.conv1) + gi * C;
            float* dc1 = prm.dconv1 + gi * C;
            float du = 0.f, dv = 0.f, dwn = 0.f;
            if (rec[CR_MASK * COST_TILE + i] != 0.f && dc != 0.f) {
                const ValueTaps vt(cost_taps(rec, i, h, w), w, c2);
                const float cn = prm.weight ? __ldg(prm.weight + gi) : 1.f;
                float t4[4], s = 0.f, r1 = 1.f;
                if constexpr (ROBUST) {
                    for (int c = lane; c < C; c += 32) { const float d = vt.residual(img, c1, c, t4); s = fmaf(d, d, s); }
                    s = warp_sum(s);
                    r1 = robust_rho1(prm.robust, prm.robust_scale, s);
                }
                const float k2 = 2.f * (dc * (cn * r1));                               // dd_c = 2 dcost c rho'(s) d_c
                float s2 = 0.f;
                for (int c = lane; c < C; c += 32) {
                    const float d = vt.residual(img, c1, c, t4);
                    const float dd = k2 * d;
                    dc1[c] = dd;
                    vt.adjoint(dimg, c, t4, -dd, du, dv);
                    if constexpr (!ROBUST) s2 = fmaf(d, d, s2);
                }
                du = warp_sum(du); dv = warp_sum(dv);
                if constexpr (!ROBUST) s = warp_sum(s2);
                dwn = dc * (ROBUST ? robust_rho(prm.robust, prm.robust_scale, s) : s);
            } else {
                for (int c = lane; c < C; c += 32) dc1[c] = 0.f;
            }
            if (lane == 0) {
                rec[CR_DU * COST_TILE + i] = du; rec[CR_DV * COST_TILE + i] = dv;
                if (prm.dweight) prm.dweight[gi] = dwn;
            }
        }
        __syncthreads();
        // ---- thread per point: geometry backward (dJ = 0) -> dD, dR, dT --------------------------------------------------------------------
        if (tid < COST_TILE) {
            const int pt = __float_as_int(rec[CR_IDX * COST_TILE + tid]);
            float gDt = 0.f;
            if (pt >= 0 && rec[CR_MASK * COST_TILE + tid] != 0.f && dc != 0.f) {
                const float* pp = prm.p + (size_t)b * 3 * N + pt;
                const float p0 = pp[0], p1 = pp[N], p2 = pp[2 * (size_t)N], Dt = rec[CR_DT * COST_TILE + tid];
                const Projection pr(sPose, p0, p1, p2, Dt);
                const float z6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                const GeomGrad gg(pr, sPose[12], sPose[13], Dt, rec[CR_DU * COST_TILE + tid], rec[CR_DV * COST_TILE + tid], z6, z6, 0.f, 0.f);
                accT[0] += gg.gX; accT[1] += gg.gY; accT[2] += gg.gZ;
                accR[0] += gg.grx * p0; accR[1] += gg.grx * p1; accR[2] += gg.grx * p2;
                accR[3] += gg.gry * p0; accR[4] += gg.gry * p1; accR[5] += gg.gry * p2;
                accR[6] += gg.grz * p0; accR[7] += gg.grz * p1; accR[8] += gg.grz * p2;
                gDt = gg.gDt;
            }
            if (pt >= 0) prm.dD[(size_t)b * N + pt] = gDt;
            rec[CR_VAL * COST_TILE + tid] = gDt;
        }
        // ---- the depth update's adjoint: dB = dDt W (one writer), dW = sum_n dDt b (column sums) --------------------------------------------
        if (KP > 0) {
            __syncthreads();
            for (int j = tid; j < COST_TILE * K; j += COST_THREADS) {
                const int i = j / K, k = j - i * K, pt = __float_as_int(rec[CR_IDX * COST_TILE + i]);
                if (pt >= 0) prm.dB[((size_t)b * N + pt) * K + k] = rec[CR_VAL * COST_TILE + i] * sW[k];
            }
            if (tid < K) {
                for (int i = 0; i < COST_TILE; ++i) accW = fmaf(rec[CR_VAL * COST_TILE + i], Bs[i * LDB + tid], accW);
            }
        }
        __syncthreads();
    }
    if (cur_b >= 0) commit(cur_b);
}

// ---- host side ------------------------------------------------------------------------------------------------------------------------------
static void cost_layout(const banet_level_t* lv, CostParams* prm)
{
    prm->nb = lv->nb; prm->N = lv->N; prm->C = lv->C; prm->K = lv->K; prm->KP = padded_K(lv->K); prm->h = lv->h; prm->w = lv->w;
    prm->grid_w = lv->grid_w; prm->grid_h = lv->grid_h;
    prm->tiles_x = lv->grid_w > 0 ? (lv->grid_w + 7) / 8 : 0;
    prm->tiles_per_pair = lv->grid_w > 0 ? prm->tiles_x * ((lv->grid_h + 7) / 8) : (lv->N + COST_TILE - 1) / COST_TILE;
    prm->total_tiles = (long long)lv->nb * prm->tiles_per_pair;
}

size_t lm_cost_ws_bytes(const banet_level_t* lv)
{
    CostParams prm;
    cost_layout(lv, &prm);
    return align_up((size_t)prm.total_tiles * 2 * sizeof(double), 256);
}

static CostParams cost_params(const banet_level_t* lv, const float* R, const float* T, const float* W)
{
    CostParams prm;
    memset(&prm, 0, sizeof(prm));
    cost_layout(lv, &prm);
    prm.conv1 = lv->conv1; prm.conv2 = lv->conv2; prm.intr = lv->intr; prm.p = lv->p; prm.D = lv->D; prm.B = lv->B;
    prm.R = R; prm.T = T; prm.W = W; prm.weight = lv->weight; prm.robust = lv->robust; prm.robust_scale = lv->robust_scale;
    const bool bf = lv->feature_dtype == BANET_DTYPE_BF16;
    prm.vec4 = (lv->C % 4 == 0) && (lv->conv2_channels % 4 == 0) &&
               ((reinterpret_cast<uintptr_t>(lv->conv1) | reinterpret_cast<uintptr_t>(lv->conv2)) % (bf ? 8 : 16) == 0);
    return prm;
}

typedef void (*CostKernel)(const CostParams);
template <template <typename, typename, bool, bool> class Pick>
static CostKernel pick_cost_kernel(const banet_level_t* lv)
{
    const bool bff = lv->feature_dtype == BANET_DTYPE_BF16, bfb = lv->K > 0 && lv->basis_dtype == BANET_DTYPE_BF16;
    const bool fly = lv->conv2_channels == lv->C, rob = lv->robust != BANET_ROBUST_NONE;
#define BANET_COST_PICK(TFV, TBV) (fly ? (rob ? Pick<TFV, TBV, true, true>::get() : Pick<TFV, TBV, true, false>::get()) \
                                       : (rob ? Pick<TFV, TBV, false, true>::get() : Pick<TFV, TBV, false, false>::get()))
    if (bff) return bfb ? BANET_COST_PICK(bf16, bf16) : BANET_COST_PICK(bf16, float);
    return bfb ? BANET_COST_PICK(float, bf16) : BANET_COST_PICK(float, float);
#undef BANET_COST_PICK
}
template <typename TF, typename TB, bool FLY, bool ROB> struct PickFwd { static CostKernel get() { return lm_cost_kernel<TF, TB, FLY, ROB>; } };
template <typename TF, typename TB, bool FLY, bool ROB> struct PickBwd { static CostKernel get() { return lm_cost_bwd_kernel<TF, TB, FLY, ROB>; } };

// persistent grid: as many CTAs as fit (at most 4 per SM), never more than there are tiles; the results do not depend on it
static int cost_launch(CostKernel kern, const CostParams& prm, cudaStream_t st, const char* what)
{
    const size_t smem = cost_smem_bytes(prm.KP);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("%s: smem attr (%zu B): %s", what, smem, cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, COST_THREADS, smem) != cudaSuccess || per_sm < 1) { cudaGetLastError(); per_sm = 1; }
    if (per_sm > 4) per_sm = 4;
    long long grid = (long long)num_sms() * per_sm;
    if (grid > prm.total_tiles) grid = prm.total_tiles;
    kern<<<(int)grid, COST_THREADS, smem, st>>>(prm);
    BANET_CUDA_LAUNCH_CHECK(what);
    return BANET_OK;
}

int launch_cost_reduce(const double* partials, int nb, int tiles_per_pair, float* cost, float* nvalid, cudaStream_t st)
{
    const long long blocks = ((long long)nb * 32 + 255) / 256;
    lm_cost_reduce_kernel<<<(unsigned)(blocks < (1LL << 20) ? blocks : (1LL << 20)), 256, 0, st>>>(partials, nb, tiles_per_pair, cost, nvalid);
    BANET_CUDA_LAUNCH_CHECK("lm_cost_reduce_kernel launch");
    return BANET_OK;
}

int lm_cost(const banet_level_t* lv, const float* R, const float* T, const float* W, float* cost, float* nvalid, float* s, float* mask,
            void* ws, cudaStream_t st)
{
    CostParams prm = cost_params(lv, R, T, W);
    prm.partials = reinterpret_cast<double*>(ws); prm.s_out = s; prm.mask_out = mask;
    int rc = cost_launch(pick_cost_kernel<PickFwd>(lv), prm, st, "lm_cost_kernel launch");
    if (rc) return rc;
    return launch_cost_reduce(prm.partials, lv->nb, prm.tiles_per_pair, cost, nvalid, st);
}

int lm_cost_bwd(const banet_level_t* lv, const float* R, const float* T, const float* W, const float* dcost, float* dconv1, float* dconv2,
                float* dD, float* dB, float* dR, float* dT, float* dW, float* dweight, cudaStream_t st)
{
    CostParams prm = cost_params(lv, R, T, W);
    prm.dcost = dcost; prm.dconv1 = dconv1; prm.dconv2 = dconv2; prm.dD = dD; prm.dB = dB; prm.dR = dR; prm.dT = dT; prm.dW = dW;
    prm.dweight = dweight;
    cudaMemsetAsync(dconv2, 0, (size_t)lv->nb * lv->h * lv->w * lv->conv2_channels * sizeof(float), st);
    cudaMemsetAsync(dR, 0, (size_t)lv->nb * 9 * sizeof(float), st);
    cudaMemsetAsync(dT, 0, (size_t)lv->nb * 3 * sizeof(float), st);
    if (lv->K > 0) cudaMemsetAsync(dW, 0, (size_t)lv->nb * lv->K * sizeof(float), st);
    return cost_launch(pick_cost_kernel<PickBwd>(lv), prm, st, "lm_cost_bwd_kernel launch");
}

}  // namespace banet
