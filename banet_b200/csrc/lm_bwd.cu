// Fused analytic backward of one LM iteration (training path of the BA layer).
//
// Forward (banet_lm_build + banet_lm_solve_update) = reference bundlenet.py:206-278 with the native op EquationConstruction (utils.cu:219-417);
// the reference differentiates that graph with TF autodiff + the registered op gradient EquationConstructionGrad (bundlenet.py:79-82,
// utils.cu:465-694), materialising J [nb,N,2,P], G, d and a tiled [nb,N,P,P] copy of the upstream gradient (utils.cu:613-617).
// Here nothing per-pixel is materialised: each pixel is re-derived from the inputs, exactly as in the forward kernels.
//
// lm_build_bwd_kernel: with Ghat = dL/dH [P,P] (as the solve's backward produces it: NOT symmetric), ghat = dL/dg, rhat = dL/drbar_sum,
//   S = 2 Ghat (the reference's op gradient, utils.cu:648) or Ghat + Ghat^T (exact adjoint), J = [Jc | jd b^T], M = G^T G, q = G^T d:
//     Y = J S              Q = Y J^T (2x2)        z = J ghat (2)
//     dJ = M Y + q ghat^T  (utils.cu:648-679)     dG_c = G_c Q + d_c z^T (:681-690)     dd_c = G_c z (:636-645) + rhat_c sign(d_c)
//   In block form the only K^2 work per pixel is e = b^T S_dd; everything else is O(K):
//     Y_c = Jc S_cc + jd (b^T S_dc)     Y_d b = Jc (S_cd b) + jd (e.b)     db = s e + S_cd^T v + t ghat_d + dDt W
//   then the chain rule through the sampler (features: atomics into dconv2; coordinates: tap differences), the projection, the
//   warp (dR, dT), and the depth update (dD, dB, dW).  With point weights (H = sum w_n H_n, g = sum w_n g_n) the Ghat / ghat adjoints of
//   pixel n are scaled by w_n and dw_n = 1/2 <M, Q> + q.z, stored by its one writer.  A robust level weighs by w_n = c_n rho'(s_n),
//   s_n = d^T d: dweight_n = dw rho'(s_n) goes to the confidence c_n, and ds = dw c_n rho''(s_n) adds 2 ds d_c to each channel's dd_c.
// pose_update_bwd_kernel: the SE(3) update's backward, thread per pair, for the dense keyframe window (lm_window.cu); the solve's backward is
//   lm_step_bwd_kernel (lm_step.cu).
#include "common.cuh"
#include "features.cuh"
#include "lm_build.h"
#include "pose_bwd.cuh"
#include "point.cuh"

namespace banet {

constexpr int BWD_THREADS = 256;
constexpr int BWD_WARPS = BWD_THREADS / 32;
constexpr int BWD_TILE = 64;
constexpr int BWD_KL_MAX = 8;                    // K <= 32 * BWD_KL_MAX

struct BwdParams {
    int nb, N, C, K, h, w;
    const void *conv1, *conv2;                   // element type: the kernel's TF (the level's feature_dtype)
    const float *intr, *p, *D;
    const void* B;                               // element type: the kernel's TB (the level's basis_dtype)
    const float *R, *T, *W;
    const float *dH, *dg, *drbar;
    float *dconv1, *dconv2, *dD, *dB, *dR, *dT, *dW;
    const float* weight;                         // [nb,N] point weights, or NULL (= 1)
    float* dweight;                              // [nb,N] their gradient, or NULL
    int exact_sym, tiles_per_pair;
    long long total_tiles;
    int robust;                                  // BANET_ROBUST_*: the weight is weight * rho'(s) (robust_rho1)
    float robust_scale;
};

// conv2 layouts of the build backward.  F2-only: the gradient channels are the forward's on-the-fly stencil at each tap,
//   gx_tau = 1/2 (F[y, rho(x+1)] - F[y, rho(x-1)]),  gy_tau = 1/2 (F[rho(y+1), x] - F[rho(y-1), x]),
// so its adjoint scatters w_tau df into the tap and +-1/2 w_tau dgx, +-1/2 w_tau dgy into the tap's four stencil neighbours (20 addresses;
// the atomics keep texels that the reflect and the clamp make coincide correct).  Summing an interior point's 20 contributions into its 12
// distinct texels first (12 atomics) was slower on an H100 at every measured size (DESIGN.md §4), so every point takes the plain scatter.
constexpr int BWD_3C = 0, BWD_F2 = 1;

// smem layout (floats): S_dd [K][K] | S_cd [6][K] | S_dc [K][6] | S_cc [36] | ghat [P] | W [K] | pose [16] | rhat [C]
// TF: feature element type (float or bf16, widened on load); dconv1 / dconv2 are fp32 for both.  TB: the same for the basis; dB is fp32.
// ROBUST: the level has a robust loss (s, rho', rho'' and the 2 ds d_c term).  A non-robust level runs the instantiation without them: its
// code is that of a library without robust losses (the robust work would otherwise stay live at this kernel's 128-register cap and spill).
template <int BWD_KL, int LAYOUT, typename TF, typename TB = float, bool ROBUST = false>
__global__ void __launch_bounds__(BWD_THREADS, 2)
lm_build_bwd_kernel(const BwdParams prm)
{
    extern __shared__ __align__(16) float sm[];
    constexpr bool FLY = LAYOUT != BWD_3C;
    const int K = prm.K, C = prm.C, N = prm.N, h = prm.h, w = prm.w, P = 6 + K, C3 = FLY ? C : 3 * C;   // C3: conv2's channel stride
    float* Sdd = sm;
    float* Scd = Sdd + (size_t)K * K;
    float* Sdc = Scd + 6 * K;
    float* Scc = Sdc + 6 * K;
    float* sg = Scc + 36;                    // ghat: [0,6) pose part, [6,P) depth part
    float* sW = sg + P;
    float* sPose = sW + K;
    float* sRh = sPose + 16;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long t_begin = part_begin(prm.total_tiles, gridDim.x, blockIdx.x);
    const long long t_end = part_begin(prm.total_tiles, gridDim.x, blockIdx.x + 1);
    int cur_b = -1;
    // per-warp accumulators of the pair-level gradients (committed with atomics at a pair change)
    float accR[9], accT[3], accW[BWD_KL];
#pragma unroll
    for (int i = 0; i < 9; ++i) accR[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) accT[i] = 0.f;
#pragma unroll
    for (int i = 0; i < BWD_KL; ++i) accW[i] = 0.f;

    auto commit = [&](int b) {
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < 9; ++i) atomicAdd(prm.dR + (size_t)b * 9 + i, accR[i]);
#pragma unroll
            for (int i = 0; i < 3; ++i) atomicAdd(prm.dT + (size_t)b * 3 + i, accT[i]);
        }
#pragma unroll
        for (int i = 0; i < BWD_KL; ++i) { const int k = lane + 32 * i; if (k < K) atomicAdd(prm.dW + (size_t)b * K + k, accW[i]); accW[i] = 0.f; }
#pragma unroll
        for (int i = 0; i < 9; ++i) accR[i] = 0.f;
#pragma unroll
        for (int i = 0; i < 3; ++i) accT[i] = 0.f;
    };

    for (long long t = t_begin; t < t_end; ++t) {
        const int b = (int)(t / prm.tiles_per_pair);
        const int n0 = (int)(t - (long long)b * prm.tiles_per_pair) * BWD_TILE;
        const int cnt = min(BWD_TILE, N - n0);
        if (b != cur_b) {
            if (cur_b >= 0) commit(cur_b);
            __syncthreads();
            const float* Gh = prm.dH + (size_t)b * P * P;
            for (int i = tid; i < P * P; i += BWD_THREADS) {
                const int r = i / P, c = i - r * P;
                const float v = prm.exact_sym ? (Gh[i] + Gh[(size_t)c * P + r]) : 2.f * Gh[i];
                if (r < 6 && c < 6) Scc[r * 6 + c] = v;
                else if (r < 6) Scd[r * K + (c - 6)] = v;
                else if (c < 6) Sdc[(r - 6) * 6 + c] = v;
                else Sdd[(size_t)(r - 6) * K + (c - 6)] = v;
            }
            for (int i = tid; i < P; i += BWD_THREADS) sg[i] = prm.dg[(size_t)b * P + i];
            for (int i = tid; i < K; i += BWD_THREADS) sW[i] = prm.W[(size_t)b * K + i];
            for (int i = tid; i < C; i += BWD_THREADS) sRh[i] = prm.drbar[(size_t)b * C + i];
            if (tid < 9) sPose[tid] = prm.R[b * 9 + tid];
            else if (tid < 12) sPose[tid] = prm.T[b * 3 + tid - 9];
            else if (tid < 16) sPose[tid] = prm.intr[b * 4 + tid - 12];
            __syncthreads();
            cur_b = b;
        }
        const float fx = sPose[12], fy = sPose[13];
        const TF* img = static_cast<const TF*>(prm.conv2) + (size_t)b * h * w * C3;
        float* dimg = prm.dconv2 + (size_t)b * h * w * C3;

        for (int pi = warp; pi < cnt; pi += BWD_WARPS) {
            const int n = n0 + pi;
            const size_t gi = (size_t)b * N + n;
            // ---- depth update and basis row (lanes over k) -----------------------------------------------------------------------
            float bl[BWD_KL];
            float bw = 0.f;
#pragma unroll
            for (int i = 0; i < BWD_KL; ++i) {
                const int k = lane + 32 * i;
                bl[i] = (k < K) ? ld_stream_elem(static_cast<const TB*>(prm.B) + gi * K + k) : 0.f;
                if (k < K) bw = fmaf(bl[i], sW[k], bw);
            }
            bw = warp_sum(bw);
            const float* pp = prm.p + (size_t)b * 3 * N + n;
            const float p0 = __ldg(pp), p1 = __ldg(pp + N), p2 = __ldg(pp + 2 * (size_t)N);
            const float Dt = __ldg(prm.D + gi) + bw;                                     // bundlenet.py:208
            const Projection pr(sPose, p0, p1, p2, Dt);
            float* dc1 = prm.dconv1 + gi * C;
            if (!pr.in_bounds(h, w)) {                   // masked pixel: no gradient at all (mask is piecewise constant)
                for (int c = lane; c < C; c += 32) dc1[c] = 0.f;
#pragma unroll
                for (int i = 0; i < BWD_KL; ++i) { const int k = lane + 32 * i; if (k < K) prm.dB[gi * K + k] = 0.f; }
                if (lane == 0) { prm.dD[gi] = 0.f; if (prm.dweight) prm.dweight[gi] = 0.f; }
                continue;
            }
            const Taps tp = taps_at(pr.u, pr.v, h, w);
            const TF* c1 = static_cast<const TF*>(prm.conv1) + gi * C;
            // ---- pass 1: M = G^T G, q = G^T d (lanes over channels) ----------------------------------------------------------------
            PointMQ mq = point_mq<FLY>(img, c1, tp, h, w, C, lane);
            // ---- Jacobians (bundlenet.py:49-74) ------------------------------------------------------------------------------------
            float a0[6], a1[6], jd0, jd1;
            camera_jacobian(fx, fy, pr.x, pr.y, pr.iZ, a0, a1);
            depth_jacobian(fx, fy, pr.rx, pr.ry, pr.rz, pr.x, pr.y, pr.iZ, jd0, jd1);
            // ---- K-dimensional contractions -----------------------------------------------------------------------------------------
            float e[BWD_KL];
            float alpha[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, beta[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, eta = 0.f, gamma = 0.f;
#pragma unroll
            for (int i = 0; i < BWD_KL; ++i) e[i] = 0.f;
            if (K > 0) {
#pragma unroll
                for (int i2 = 0; i2 < BWD_KL; ++i2) {                          // e = b^T S_dd  (b_j broadcast from the lane that holds it)
                    if (32 * i2 >= K) break;
#pragma unroll 2
                    for (int j2 = 0; j2 < 32; ++j2) {
                        const int j = 32 * i2 + j2;
                        if (j >= K) break;
                        const float bj = __shfl_sync(0xffffffffu, bl[i2], j2);
                        const float* row = Sdd + (size_t)j * K;
#pragma unroll
                        for (int i = 0; i < BWD_KL; ++i) { const int k = lane + 32 * i; if (k < K) e[i] = fmaf(bj, row[k], e[i]); }
                    }
                }
#pragma unroll
                for (int i = 0; i < BWD_KL; ++i) {
                    const int k = lane + 32 * i;
                    if (k < K) {
                        gamma = fmaf(e[i], bl[i], gamma); eta = fmaf(sg[6 + k], bl[i], eta);
#pragma unroll
                        for (int m = 0; m < 6; ++m) { alpha[m] = fmaf(Scd[m * K + k], bl[i], alpha[m]); beta[m] = fmaf(Sdc[k * 6 + m], bl[i], beta[m]); }
                    }
                }
                gamma = warp_sum(gamma); eta = warp_sum(eta);
#pragma unroll
                for (int m = 0; m < 6; ++m) { alpha[m] = warp_sum(alpha[m]); beta[m] = warp_sum(beta[m]); }
            }
            // ---- 2 x (6+1) algebra (every lane, redundantly), the point weight, dJ and the depth terms of db --------------------------
            PointAdjoint ad(a0, a1, jd0, jd1, Scc, sg, alpha, beta, eta, gamma);
            const float cn = prm.weight ? __ldg(prm.weight + gi) : 1.f;
            float r1 = 1.f, r2 = 0.f, ds2 = 0.f;
            if constexpr (ROBUST) r1 = robust_rho1(prm.robust, prm.robust_scale, warp_sum(mq.s), &r2);
            const float dw = ad.weigh(ROBUST ? cn * r1 : cn, mq);
            if (prm.dweight && lane == 0) prm.dweight[gi] = ROBUST ? dw * r1 : dw;
            if constexpr (ROBUST) ds2 = 2.f * (dw * cn * r2);                          // 2 ds: the robust weight's share of each channel's dd_c
            float dJ0[6], dJ1[6], dj0, dj1, vN[8];                 // depth terms of db: vN (6), then tN, sN
            jacobian_adjoint(mq, ad, sg, eta, dJ0, dJ1, dj0, dj1);
            depth_terms(a0, a1, jd0, jd1, mq, vN);
            const float tN = vN[6], sN = vN[7];
            // ---- pass 2: dd, dG per channel -> dconv1, scatter into dconv2, coordinate gradient ------------------------------------------
            float du, dv;
            channel_adjoint<FLY>(img, dimg, c1, sRh, tp, h, w, C, lane, ad, ds2, [&](int c, float dd) { dc1[c] = dd; }, du, dv);
            // ---- geometry backward ----------------------------------------------------------------------------------------------------
            const GeomGrad gg(pr, fx, fy, Dt, du, dv, dJ0, dJ1, dj0, dj1);
            accT[0] += gg.gX; accT[1] += gg.gY; accT[2] += gg.gZ;
            accR[0] += gg.grx * p0; accR[1] += gg.grx * p1; accR[2] += gg.grx * p2;
            accR[3] += gg.gry * p0; accR[4] += gg.gry * p1; accR[5] += gg.gry * p2;
            accR[6] += gg.grz * p0; accR[7] += gg.grz * p1; accR[8] += gg.grz * p2;
            if (lane == 0) prm.dD[gi] = gg.gDt;
            // ---- dB row, dW ---------------------------------------------------------------------------------------------------------
#pragma unroll
            for (int i = 0; i < BWD_KL; ++i) {
                const int k = lane + 32 * i;
                if (k < K) {
                    float db = sN * e[i] + tN * sg[6 + k] + gg.gDt * sW[k];
#pragma unroll
                    for (int m = 0; m < 6; ++m) db = fmaf(vN[m], Scd[m * K + k], db);
                    prm.dB[gi * K + k] = db;
                    accW[i] = fmaf(gg.gDt, bl[i], accW[i]);
                }
            }
        }
    }
    if (cur_b >= 0) commit(cur_b);
}

template <typename TF, typename TB, bool R>
static void (*select_bwd_kernel_r(int K, bool c3))(const BwdParams)
{
    if (c3) return K <= 32 ? lm_build_bwd_kernel<1, BWD_3C, TF, TB, R> : (K <= 128 ? lm_build_bwd_kernel<4, BWD_3C, TF, TB, R> : lm_build_bwd_kernel<8, BWD_3C, TF, TB, R>);
    return K <= 32 ? lm_build_bwd_kernel<1, BWD_F2, TF, TB, R> : (K <= 128 ? lm_build_bwd_kernel<4, BWD_F2, TF, TB, R> : lm_build_bwd_kernel<8, BWD_F2, TF, TB, R>);
}
template <typename TF, typename TB>
static void (*select_bwd_kernel(int K, bool c3, bool robust))(const BwdParams)
{
    return robust ? select_bwd_kernel_r<TF, TB, true>(K, c3) : select_bwd_kernel_r<TF, TB, false>(K, c3);
}

int lm_build_bwd(const banet_level_t* lv, const float* R, const float* T, const float* W, const float* dH, const float* dg, const float* drbar,
                 int exact_sym, float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW, float* dweight, cudaStream_t st)
{
    const int K = lv->K, P = 6 + K;
    BANET_REQUIRE(K <= 32 * BWD_KL_MAX, BANET_ERR_UNSUPPORTED, "lm_build_bwd: K=%d > %d", K, 32 * BWD_KL_MAX);
    const size_t smem = ((size_t)K * K + 12 * (size_t)K + 36 + P + K + 16 + lv->C) * sizeof(float);
    BANET_REQUIRE(smem <= 220 * 1024, BANET_ERR_UNSUPPORTED, "lm_build_bwd: K=%d, C=%d need %zu B of shared memory", K, lv->C, smem);
    void (*kern)(const BwdParams);
    const bool c3 = lv->conv2_channels == 3 * lv->C, bff = lv->feature_dtype == BANET_DTYPE_BF16, bfb = K > 0 && lv->basis_dtype == BANET_DTYPE_BF16;
    const bool rob = lv->robust != BANET_ROBUST_NONE;
    if (bfb) kern = bff ? select_bwd_kernel<bf16, bf16>(K, c3, rob) : select_bwd_kernel<float, bf16>(K, c3, rob);
    else kern = bff ? select_bwd_kernel<bf16, float>(K, c3, rob) : select_bwd_kernel<float, float>(K, c3, rob);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("lm_build_bwd smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    BwdParams prm;
    prm.nb = lv->nb; prm.N = lv->N; prm.C = lv->C; prm.K = K; prm.h = lv->h; prm.w = lv->w;
    prm.conv1 = lv->conv1; prm.conv2 = lv->conv2; prm.intr = lv->intr; prm.p = lv->p; prm.D = lv->D; prm.B = lv->B; prm.R = R; prm.T = T; prm.W = W;
    prm.dH = dH; prm.dg = dg; prm.drbar = drbar;
    prm.dconv1 = dconv1; prm.dconv2 = dconv2; prm.dD = dD; prm.dB = dB; prm.dR = dR; prm.dT = dT; prm.dW = dW;
    prm.weight = lv->weight; prm.dweight = dweight;
    prm.robust = lv->robust; prm.robust_scale = lv->robust_scale;
    prm.exact_sym = exact_sym;
    prm.tiles_per_pair = (lv->N + BWD_TILE - 1) / BWD_TILE;
    prm.total_tiles = (long long)lv->nb * prm.tiles_per_pair;
    cudaMemsetAsync(dconv2, 0, (size_t)lv->nb * lv->h * lv->w * lv->conv2_channels * sizeof(float), st);
    cudaMemsetAsync(dR, 0, (size_t)lv->nb * 9 * sizeof(float), st);
    cudaMemsetAsync(dT, 0, (size_t)lv->nb * 3 * sizeof(float), st);
    if (K > 0) cudaMemsetAsync(dW, 0, (size_t)lv->nb * K * sizeof(float), st);
    int per_sm = (int)((220 * 1024) / (smem + 1024)); if (per_sm < 1) per_sm = 1; if (per_sm > 2) per_sm = 2;
    long long grid = (long long)num_sms() * per_sm;
    if (grid > prm.total_tiles) grid = prm.total_tiles;
    kern<<<(int)grid, BWD_THREADS, smem, st>>>(prm);
    BANET_CUDA_LAUNCH_CHECK("lm_build_bwd_kernel launch");
    return BANET_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------------
// SE(3) update backward
// ------------------------------------------------------------------------------------------------------------------------------------
// SE(3) update backward, thread per pair, double (R' = exp(w) R, T' = V(w) t + exp(w) T; bundlenet.py:269-275): writes
// ddelta[0:6] (into `ddelta`, row stride P), dR, dT.
__global__ void pose_update_bwd_kernel(const float* __restrict__ delta, int nb, int P, const float* __restrict__ R, const float* __restrict__ T,
                                       const float* __restrict__ gRn, const float* __restrict__ gTn,
                                       float* __restrict__ ddelta, float* __restrict__ dR, float* __restrict__ dT)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    double dl[6];
    for (int i = 0; i < 6; ++i) { dl[i] = delta[(size_t)b * P + i]; if (!isfinite(dl[i])) dl[i] = 0.0; }
    pose_update_bwd_one(dl, R + (size_t)b * 9, T + (size_t)b * 3, gRn + (size_t)b * 9, gTn + (size_t)b * 3, ddelta + (size_t)b * P, dR + (size_t)b * 9, dT + (size_t)b * 3);
}

int launch_pose_update_bwd(const float* delta, int nb, int P, const float* R, const float* T, const float* gRn, const float* gTn,
                           float* ddelta, float* dR, float* dT, cudaStream_t st)
{
    pose_update_bwd_kernel<<<(nb + 63) / 64, 64, 0, st>>>(delta, nb, P, R, T, gRn, gTn, ddelta, dR, dT);
    BANET_CUDA_LAUNCH_CHECK("pose_update_bwd_kernel launch");
    return BANET_OK;
}

}  // namespace banet
