// Feature-metric cost of keyframe windows and its backward (include/banet_abi.h section 3e, banet_lm_keyframe_cost / _bwd): banet_lm_cost
// on the keyframe layout, the keyframe's tensors once per window.  Pair b = w nf + f samples keyframe point n of window w at
//
//   s_{b,n} = sum_c d^2,  d = conv1[w,n] - F2_b(pi(p[w,n], D[w,n] + B[w,n].W_w; R_b, T_b)),   cost[b] = sum_n c_{b,n} s_{b,n} (in-bounds n)
//
// with lm_cost.cu's per-point arithmetic (cost_tile.cuh, point.cuh), so every output equals banet_lm_cost's on the keyframe replicated
// per frame, bit for bit.  fp32 only, no robust loss (the keyframe layout has neither); conv2 is [F2|gx|gy] or F2 only (c2 at run time).
//
// keyframe_cost_kernel: persistent over the nw ceil(N/64) keyframe tiles of 64 consecutive points.  Per tile: stage the basis rows and
//   D + b.W_w once (lm_cost_kernel's S0 / S1 arithmetic), then walk the frames in order: thread per point the projection, mask and taps;
//   warp per point the value taps of every channel (cost_point_s); one warp sums the tile in fp64 (cost_tile_sum) into slot (w nf + f, tile).
//   The slots are laid out [pair][tile] as lm_cost_kernel's, so lm_cost_reduce_kernel sums them unchanged (launch_cost_reduce).
// keyframe_cost_bwd_kernel: the same tiles and staging; then warp per keyframe point with the frames walked inside the point, in chunks of
//   KC_FRAMES.  Per frame: dd = 2 dcost_b c d into the point's running dconv1 row (shared memory), ValueTaps::adjoint into pair b's dconv2
//   (atomics), GeomGrad with dJ = 0 into the warp's per-frame dR, dT sums and the point's running dDt.  dconv1 is stored after every chunk
//   and re-read by the next (one writer: point n's warp), dD after the last; then dB = dDt W_w (one writer) and dW_w = sum_n dDt b in
//   per-column sums, committed with atomics at a window change.  Every frame sum is taken in frame order: bit-reproducible.
#include "common.cuh"
#include "cost_tile.cuh"
#include "lm_build.h"
#include "point.cuh"
#include <string.h>

namespace banet {
namespace {

constexpr int KC_FRAMES = 16;                    // backward: frames per chunk of the per-warp dR, dT sums

struct KeyCostParams {
    int nw, nf, N, C, K, KP, h, w, c2, vec4, tiles_per_win;
    long long total_tiles;
    const float *conv1, *p, *D, *B;              // keyframe, [nw,...]
    const float *conv2, *intr, *R, *T;           // per pair, [nw nf,...]
    const float *W, *weight;                     // [nw,K]; [nw nf,N] or NULL (= 1)
    double* partials;                            // forward: [nw nf][tiles_per_win][2] = (sum c s, in-bounds count) per (pair, tile)
    float *s_out, *mask_out;                     // forward, optional
    const float* dcost;                          // backward
    float *dconv1, *dconv2, *dD, *dB, *dR, *dT, *dW, *dweight;
};

// smem (floats): Bs [64][KP+4] | W [KP] | pose [16] | rays [3][64] | records [CR_ARRAYS][64]
//   backward, then: dconv1 row per warp [COST_WARPS][C] | dR, dT per warp and frame of the chunk [COST_WARPS][KC_FRAMES][12]
static size_t key_cost_smem_floats(int KP) { return (size_t)COST_TILE * (KP + 4) + KP + 16 + 3 * COST_TILE + CR_ARRAYS * COST_TILE; }
static size_t key_cost_bwd_smem_floats(int KP, int C) { return key_cost_smem_floats(KP) + (size_t)COST_WARPS * C + COST_WARPS * KC_FRAMES * 12; }

// stage keyframe tile r of window wi: the point indices, the basis rows (coalesced), and per point (thread) its ray and depth D + b.W_w in
// basis_dot's arithmetic, as lm_cost_kernel's S0 / S1 (so the mask is banet_lm_cost's and the build's); CR_VAL is cleared
__device__ __forceinline__ void key_cost_stage(const KeyCostParams& prm, int wi, int r, float* Bs, const float* sW, float* sRay, float* rec)
{
    const int tid = threadIdx.x, K = prm.K, KP = prm.KP, LDB = KP + 4, N = prm.N;
    if (tid < COST_TILE) { const int n = r * COST_TILE + tid; rec[CR_IDX * COST_TILE + tid] = __int_as_float(n < N ? n : -1); }
    __syncthreads();
    const float* Bg = prm.B + (size_t)wi * N * K;
    if ((K & 3) == 0) {
        const int k4 = K >> 2, kp4 = KP >> 2;
        for (int i = tid; i < COST_TILE * kp4; i += COST_THREADS) {
            const int n = i / kp4, q = i - n * kp4, pt = __float_as_int(rec[CR_IDX * COST_TILE + n]);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (pt >= 0 && q < k4) v = ld_stream_f4(Bg + (size_t)pt * K + 4 * q);
            *reinterpret_cast<float4*>(Bs + n * LDB + 4 * q) = v;
        }
    } else {
        for (int i = tid; i < COST_TILE * KP; i += COST_THREADS) {
            const int n = i / KP, k = i - n * KP, pt = __float_as_int(rec[CR_IDX * COST_TILE + n]);
            Bs[n * LDB + k] = (pt >= 0 && k < K) ? ld_stream_f1(Bg + (size_t)pt * K + k) : 0.f;
        }
    }
    __syncthreads();
    if (tid < COST_TILE) {
        const int pt = __float_as_int(rec[CR_IDX * COST_TILE + tid]);
        float p0 = 0.f, p1 = 0.f, p2 = 0.f, Dt = 0.f;
        if (pt >= 0) {
            const float* pp = prm.p + (size_t)wi * 3 * N + pt;
            p0 = pp[0]; p1 = pp[N]; p2 = pp[2 * (size_t)N];
            Dt = prm.D[(size_t)wi * N + pt];
            Dt += basis_dot_padded(Bs + tid * LDB, sW, KP);
        }
        sRay[tid] = p0; sRay[COST_TILE + tid] = p1; sRay[2 * COST_TILE + tid] = p2;
        rec[CR_DT * COST_TILE + tid] = Dt; rec[CR_VAL * COST_TILE + tid] = 0.f;
    }
    __syncthreads();
}

__device__ __forceinline__ void key_cost_window_w(const KeyCostParams& prm, int wi, float* sW)
{
    for (int k = threadIdx.x; k < prm.KP; k += COST_THREADS) sW[k] = (k < prm.K) ? prm.W[(size_t)wi * prm.K + k] : 0.f;
}

__global__ void __launch_bounds__(COST_THREADS, 4)
keyframe_cost_kernel(const KeyCostParams prm)
{
    extern __shared__ __align__(16) float smem[];
    const int KP = prm.KP;
    float* Bs = smem;
    float* sW = Bs + COST_TILE * (KP + 4);
    float* sPose = sW + KP;
    float* sRay = sPose + 16;
    float* rec = sRay + 3 * COST_TILE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = prm.N, C = prm.C, h = prm.h, w = prm.w, c2 = prm.c2, nf = prm.nf;
    const long long t_begin = part_begin(prm.total_tiles, gridDim.x, blockIdx.x);
    const long long t_end = part_begin(prm.total_tiles, gridDim.x, blockIdx.x + 1);
    int cur_w = -1;
    for (long long t = t_begin; t < t_end; ++t) {
        const int wi = (int)(t / prm.tiles_per_win), r = (int)(t - (long long)wi * prm.tiles_per_win);
        if (wi != cur_w) { key_cost_window_w(prm, wi, sW); cur_w = wi; }    // the last readers passed the previous tile's barriers
        key_cost_stage(prm, wi, r, Bs, sW, sRay, rec);
        const float* c1w = prm.conv1 + (size_t)wi * N * C;
        for (int f = 0; f < nf; ++f) {
            const size_t b = (size_t)wi * nf + f;
            if (tid < 9) sPose[tid] = prm.R[b * 9 + tid];
            else if (tid < 12) sPose[tid] = prm.T[b * 3 + tid - 9];
            else if (tid < 16) sPose[tid] = prm.intr[b * 4 + tid - 12];
            __syncthreads();                                             // also: the previous frame's S3 is done with the records
            // ---- thread per point: projection, mask, taps (lm_cost_kernel's S1) ----------------------------------------------------------
            if (tid < COST_TILE) {
                const int pt = __float_as_int(rec[CR_IDX * COST_TILE + tid]);
                float mask = 0.f, dx = 0.f, dy = 0.f;
                int x0 = 0, y0 = 0;
                if (pt >= 0) {
                    const Projection pr(sPose, sRay[tid], sRay[COST_TILE + tid], sRay[2 * COST_TILE + tid], rec[CR_DT * COST_TILE + tid]);
                    if (pr.in_bounds(h, w)) {
                        mask = 1.f;
                        tap_corner(pr.u, pr.v, x0, y0, dx, dy);
                    }
                }
                rec[CR_X0 * COST_TILE + tid] = __int_as_float(x0); rec[CR_Y0 * COST_TILE + tid] = __int_as_float(y0);
                rec[CR_DX * COST_TILE + tid] = dx; rec[CR_DY * COST_TILE + tid] = dy; rec[CR_MASK * COST_TILE + tid] = mask;
            }
            __syncthreads();
            // ---- S2: warp per point, lanes over channels -----------------------------------------------------------------------------------
            const float* img = prm.conv2 + b * h * w * c2;
            for (int i = warp; i < COST_TILE; i += COST_WARPS) {
                const int pt = __float_as_int(rec[CR_IDX * COST_TILE + i]);
                if (pt < 0) { if (lane == 0) rec[CR_VAL * COST_TILE + i] = 0.f; continue; }
                const size_t gi = b * N + pt;
                float val = 0.f, s = 0.f;
                if (rec[CR_MASK * COST_TILE + i] != 0.f) {
                    s = cost_point_s<float>(img, c1w + (size_t)pt * C, rec, i, h, w, c2, C, prm.vec4, lane);
                    const float cn = prm.weight ? __ldg(prm.weight + gi) : 1.f;
                    val = cn * s;
                }
                if (lane == 0) {
                    rec[CR_VAL * COST_TILE + i] = val;
                    if (prm.s_out) prm.s_out[gi] = s;
                    if (prm.mask_out) prm.mask_out[gi] = rec[CR_MASK * COST_TILE + i];
                }
            }
            __syncthreads();
            // ---- S3: the tile's sum for pair b, slot (b, r) ---------------------------------------------------------------------------------
            if (warp == 0) cost_tile_sum(rec, lane, prm.partials + 2 * ((long long)b * prm.tiles_per_win + r));
        }
        // the next tile's stage rewrites only what S3 does not read before its first barrier
    }
}

__global__ void __launch_bounds__(COST_THREADS, 2)
keyframe_cost_bwd_kernel(const KeyCostParams prm)
{
    extern __shared__ __align__(16) float smem[];
    const int KP = prm.KP, K = prm.K, LDB = KP + 4;
    float* Bs = smem;
    float* sW = Bs + COST_TILE * LDB;
    float* sRay = sW + KP + 16;
    float* rec = sRay + 3 * COST_TILE;
    float* sDc1 = rec + CR_ARRAYS * COST_TILE;
    float* sRT = sDc1 + (size_t)COST_WARPS * prm.C;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = prm.N, C = prm.C, h = prm.h, w = prm.w, c2 = prm.c2, nf = prm.nf;
    float* myDc1 = sDc1 + (size_t)warp * C;
    const long long t_begin = part_begin(prm.total_tiles, gridDim.x, blockIdx.x);
    const long long t_end = part_begin(prm.total_tiles, gridDim.x, blockIdx.x + 1);
    const float z6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int cur_w = -1;
    float accW = 0.f;                                                    // dW column tid of the current window (tid < K)
    for (long long t = t_begin; t < t_end; ++t) {
        const int wi = (int)(t / prm.tiles_per_win), r = (int)(t - (long long)wi * prm.tiles_per_win);
        if (wi != cur_w) {
            if (cur_w >= 0 && tid < K) atomicAdd(prm.dW + (size_t)cur_w * K + tid, accW);
            accW = 0.f;
            key_cost_window_w(prm, wi, sW);
            cur_w = wi;
        }
        key_cost_stage(prm, wi, r, Bs, sW, sRay, rec);
        for (int fc0 = 0; fc0 < nf; fc0 += KC_FRAMES) {
            const int nfl = min(KC_FRAMES, nf - fc0);
            const bool last = fc0 + nfl == nf;
            for (int i = tid; i < COST_WARPS * KC_FRAMES * 12; i += COST_THREADS) sRT[i] = 0.f;
            __syncthreads();
            // ---- warp per keyframe point, the chunk's frames in order inside it ------------------------------------------------------------
            for (int i = warp; i < COST_TILE; i += COST_WARPS) {
                const int pt = __float_as_int(rec[CR_IDX * COST_TILE + i]);
                if (pt < 0) continue;
                const size_t gi = (size_t)wi * N + pt;
                const float p0 = sRay[i], p1 = sRay[COST_TILE + i], p2 = sRay[2 * COST_TILE + i], Dt = rec[CR_DT * COST_TILE + i];
                const float* c1 = prm.conv1 + gi * C;
                float* dc1 = prm.dconv1 + gi * C;
                for (int c = lane; c < C; c += 32) myDc1[c] = (fc0 > 0) ? dc1[c] : 0.f;
                __syncwarp();
                float dDacc = rec[CR_VAL * COST_TILE + i];
                for (int fl = 0; fl < nfl; ++fl) {
                    const size_t b = (size_t)wi * nf + fc0 + fl;
                    const float dc = __ldg(prm.dcost + b);
                    float pose[16];
#pragma unroll
                    for (int q = 0; q < 9; ++q) pose[q] = __ldg(prm.R + b * 9 + q);
#pragma unroll
                    for (int q = 0; q < 3; ++q) pose[9 + q] = __ldg(prm.T + b * 3 + q);
#pragma unroll
                    for (int q = 0; q < 4; ++q) pose[12 + q] = __ldg(prm.intr + b * 4 + q);
                    const Projection pr(pose, p0, p1, p2, Dt);
                    if (!pr.in_bounds(h, w) || dc == 0.f) {                  // no gradient through this frame
                        if (prm.dweight && lane == 0) prm.dweight[b * N + pt] = 0.f;
                        continue;
                    }
                    const ValueTaps vt(taps_at(pr.u, pr.v, h, w), w, c2);
                    const float cn = prm.weight ? __ldg(prm.weight + b * N + pt) : 1.f;
                    const float k2 = 2.f * (dc * cn);                         // dd_c = 2 dcost c d_c
                    const float* img = prm.conv2 + b * h * w * c2;
                    float* dimg = prm.dconv2 + b * h * w * c2;
                    float t4[4], du = 0.f, dv = 0.f, s2 = 0.f;
                    for (int c = lane; c < C; c += 32) {
                        const float d = vt.residual(img, c1, c, t4);
                        const float dd = k2 * d;
                        myDc1[c] += dd;
                        vt.adjoint(dimg, c, t4, -dd, du, dv);
                        s2 = fmaf(d, d, s2);
                    }
                    du = warp_sum(du); dv = warp_sum(dv);
                    const float s = warp_sum(s2);
                    const GeomGrad gg(pr, pose[12], pose[13], Dt, du, dv, z6, z6, 0.f, 0.f);
                    if (lane == 0) {
                        if (prm.dweight) prm.dweight[b * N + pt] = dc * s;
                        float* rt = sRT + (warp * KC_FRAMES + fl) * 12;
                        rt[0] += gg.grx * p0; rt[1] += gg.grx * p1; rt[2] += gg.grx * p2;
                        rt[3] += gg.gry * p0; rt[4] += gg.gry * p1; rt[5] += gg.gry * p2;
                        rt[6] += gg.grz * p0; rt[7] += gg.grz * p1; rt[8] += gg.grz * p2;
                        rt[9] += gg.gX; rt[10] += gg.gY; rt[11] += gg.gZ;
                    }
                    dDacc += gg.gDt;
                }
                __syncwarp();
                for (int c = lane; c < C; c += 32) dc1[c] = myDc1[c];
                if (lane == 0) {
                    rec[CR_VAL * COST_TILE + i] = dDacc;
                    if (last) prm.dD[gi] = dDacc;
                }
                __syncwarp();
            }
            __syncthreads();
            // ---- commit the chunk's dR, dT: the warps' sums in a fixed order, one atomic per (pair, entry) -------------------------------------
            for (int i = tid; i < nfl * 12; i += COST_THREADS) {
                const int fl = i / 12, q = i - fl * 12;
                float s = 0.f;
                for (int wq = 0; wq < COST_WARPS; ++wq) s += sRT[(wq * KC_FRAMES + fl) * 12 + q];
                const size_t b = (size_t)wi * nf + fc0 + fl;
                if (q < 9) atomicAdd(prm.dR + b * 9 + q, s); else atomicAdd(prm.dT + b * 3 + q - 9, s);
            }
            __syncthreads();
        }
        // ---- the depth update's adjoint: dB = dDt W_w (one writer), dW_w = sum_n dDt b (column sums; masked rows carry dDt = 0) --------------
        for (int j = tid; j < COST_TILE * K; j += COST_THREADS) {
            const int i = j / K, k = j - i * K, pt = __float_as_int(rec[CR_IDX * COST_TILE + i]);
            if (pt >= 0) prm.dB[((size_t)wi * N + pt) * K + k] = rec[CR_VAL * COST_TILE + i] * sW[k];
        }
        if (tid < K) {
            for (int i = 0; i < COST_TILE; ++i) accW = fmaf(rec[CR_VAL * COST_TILE + i], Bs[i * LDB + tid], accW);
        }
        __syncthreads();
    }
    if (cur_w >= 0 && tid < K) atomicAdd(prm.dW + (size_t)cur_w * K + tid, accW);
}

// ---- host side ------------------------------------------------------------------------------------------------------------------------------
KeyCostParams key_cost_params(const banet_keyframe_level_t* lv, const float* R, const float* T, const float* W)
{
    KeyCostParams prm;
    memset(&prm, 0, sizeof(prm));
    prm.nw = lv->nw; prm.nf = lv->nf; prm.N = lv->N; prm.C = lv->C; prm.K = lv->K; prm.KP = padded_K(lv->K); prm.h = lv->h; prm.w = lv->w;
    prm.c2 = lv->conv2_channels;
    prm.tiles_per_win = (lv->N + COST_TILE - 1) / COST_TILE;
    prm.total_tiles = (long long)lv->nw * prm.tiles_per_win;
    prm.conv1 = lv->conv1; prm.p = lv->p; prm.D = lv->D; prm.B = lv->B; prm.conv2 = lv->conv2; prm.intr = lv->intr;
    prm.R = R; prm.T = T; prm.W = W; prm.weight = lv->weight;
    prm.vec4 = (lv->C % 4 == 0) && (lv->conv2_channels % 4 == 0) &&
               ((reinterpret_cast<uintptr_t>(lv->conv1) | reinterpret_cast<uintptr_t>(lv->conv2)) % 16 == 0);
    return prm;
}

// persistent grid: as many CTAs as fit (at most 4 per SM), never more than there are tiles; the results do not depend on it
int key_cost_launch(void (*kern)(const KeyCostParams), const KeyCostParams& prm, size_t smem, cudaStream_t st, const char* what)
{
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

}  // namespace

size_t keyframe_cost_ws_bytes(const banet_keyframe_level_t* lv)
{
    const long long tiles = (long long)lv->nw * lv->nf * ((lv->N + COST_TILE - 1) / COST_TILE);
    return align_up((size_t)tiles * 2 * sizeof(double), 256);
}

int keyframe_cost(const banet_keyframe_level_t* lv, const float* R, const float* T, const float* W, float* cost, float* nvalid, float* s,
                  float* mask, void* ws, cudaStream_t st)
{
    KeyCostParams prm = key_cost_params(lv, R, T, W);
    prm.partials = reinterpret_cast<double*>(ws); prm.s_out = s; prm.mask_out = mask;
    int rc = key_cost_launch(keyframe_cost_kernel, prm, key_cost_smem_floats(prm.KP) * sizeof(float), st, "keyframe_cost_kernel launch");
    if (rc) return rc;
    return launch_cost_reduce(prm.partials, lv->nw * lv->nf, prm.tiles_per_win, cost, nvalid, st);
}

int keyframe_cost_bwd(const banet_keyframe_level_t* lv, const float* R, const float* T, const float* W, const float* dcost, float* dconv1,
                      float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW, float* dweight, cudaStream_t st)
{
    KeyCostParams prm = key_cost_params(lv, R, T, W);
    prm.dcost = dcost; prm.dconv1 = dconv1; prm.dconv2 = dconv2; prm.dD = dD; prm.dB = dB; prm.dR = dR; prm.dT = dT; prm.dW = dW;
    prm.dweight = dweight;
    const size_t nb = (size_t)lv->nw * lv->nf;
    cudaMemsetAsync(dconv2, 0, nb * lv->h * lv->w * lv->conv2_channels * sizeof(float), st);
    cudaMemsetAsync(dR, 0, nb * 9 * sizeof(float), st);
    cudaMemsetAsync(dT, 0, nb * 3 * sizeof(float), st);
    cudaMemsetAsync(dW, 0, (size_t)lv->nw * lv->K * sizeof(float), st);
    return key_cost_launch(keyframe_cost_bwd_kernel, prm, key_cost_bwd_smem_floats(prm.KP, prm.C) * sizeof(float), st,
                           "keyframe_cost_bwd_kernel launch");
}

}  // namespace banet
