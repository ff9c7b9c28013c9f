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
//   warp (dR, dT), and the depth update (dD, dB, dW).
// lm_solve_update_bwd_kernel: delta = Ht^-1 g, Ht = H + diag(damp (diag H + eps)) lambda  ->  u = Ht^-1 ddelta, dg = u, dHt = -u delta^T,
//   dH = dHt (1 + damp lambda on the diagonal), dlambda = sum_i dHt_ii damp_i (H_ii + eps); ddelta from the SE(3) update by forward-mode
//   dual numbers over the same expressions as pose_update_kernel (lm_solve.cu).
#include "common.cuh"
#include "lm_build.h"
#include "pose_bwd.cuh"

namespace banet {

constexpr int BWD_THREADS = 256;
constexpr int BWD_WARPS = BWD_THREADS / 32;
constexpr int BWD_TILE = 64;
constexpr int BWD_KL_MAX = 8;                    // K <= 32 * BWD_KL_MAX

struct BwdParams {
    int nb, N, C, K, h, w;
    const float *conv1, *conv2, *intr, *p, *D, *B, *R, *T, *W;
    const float *dH, *dg, *drbar;
    float *dconv1, *dconv2, *dD, *dB, *dR, *dT, *dW;
    int exact_sym, tiles_per_pair;
    long long total_tiles;
};

__device__ __forceinline__ float sgnf(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }

// smem layout (floats): S_dd [K][K] | S_cd [6][K] | S_dc [K][6] | S_cc [36] | ghat [P] | W [K] | pose [16] | rhat [C]
template <int BWD_KL>
__global__ void __launch_bounds__(BWD_THREADS, 2)
lm_build_bwd_kernel(const BwdParams prm)
{
    extern __shared__ __align__(16) float sm[];
    const int K = prm.K, C = prm.C, N = prm.N, h = prm.h, w = prm.w, P = 6 + K, C3 = 3 * C;
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
        const float fx = sPose[12], fy = sPose[13], ox = sPose[14], oy = sPose[15];
        const float* img = prm.conv2 + (size_t)b * h * w * C3;
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
                bl[i] = (k < K) ? ld_stream_f1(prm.B + gi * K + k) : 0.f;
                if (k < K) bw = fmaf(bl[i], sW[k], bw);
            }
            bw = warp_sum(bw);
            const float* pp = prm.p + (size_t)b * 3 * N + n;
            const float p0 = __ldg(pp), p1 = __ldg(pp + N), p2 = __ldg(pp + 2 * (size_t)N);
            const float Dt = __ldg(prm.D + gi) + bw;                                     // bundlenet.py:208
            const float rx = sPose[0] * p0 + sPose[1] * p1 + sPose[2] * p2;
            const float ry = sPose[3] * p0 + sPose[4] * p1 + sPose[5] * p2;
            const float rz = sPose[6] * p0 + sPose[7] * p1 + sPose[8] * p2;
            const float X = rx * Dt + sPose[9], Y = ry * Dt + sPose[10], Z = rz * Dt + sPose[11];
            const float x = X / Z, y = Y / Z, iZ = 1.0f / Z;
            const float u = fx * x + ox, v = fy * y + oy;
            const bool ok = (u >= 0.f) && (u <= (float)(w - 1)) && (v >= 0.f) && (v <= (float)(h - 1)) && isfinite(iZ);
            float* dc1 = prm.dconv1 + gi * C;
            if (!ok) {                                   // masked pixel: no gradient at all (mask is piecewise constant)
                for (int c = lane; c < C; c += 32) dc1[c] = 0.f;
#pragma unroll
                for (int i = 0; i < BWD_KL; ++i) { const int k = lane + 32 * i; if (k < K) prm.dB[gi * K + k] = 0.f; }
                if (lane == 0) prm.dD[gi] = 0.f;
                continue;
            }
            const float fu = floorf(u), fv = floorf(v);
            const int x0 = (int)fu, y0 = (int)fv, x1 = min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1);
            const float dx = u - fu, dy = v - fv;
            const float w00 = (1.f - dx) * (1.f - dy), w01 = dx * (1.f - dy), w10 = (1.f - dx) * dy, w11 = dx * dy;
            const size_t o00 = ((size_t)y0 * w + x0) * C3, o01 = ((size_t)y0 * w + x1) * C3, o10 = ((size_t)y1 * w + x0) * C3, o11 = ((size_t)y1 * w + x1) * C3;
            const float* c1 = prm.conv1 + gi * C;
            // ---- pass 1: M = G^T G, q = G^T d (lanes over channels) ----------------------------------------------------------------
            float m11 = 0.f, m12 = 0.f, m22 = 0.f, q1 = 0.f, q2 = 0.f;
            for (int c = lane; c < C; c += 32) {
                const float f2 = w00 * __ldg(img + o00 + c) + w01 * __ldg(img + o01 + c) + w10 * __ldg(img + o10 + c) + w11 * __ldg(img + o11 + c);
                const float gx = w00 * __ldg(img + o00 + C + c) + w01 * __ldg(img + o01 + C + c) + w10 * __ldg(img + o10 + C + c) + w11 * __ldg(img + o11 + C + c);
                const float gy = w00 * __ldg(img + o00 + 2 * C + c) + w01 * __ldg(img + o01 + 2 * C + c) + w10 * __ldg(img + o10 + 2 * C + c) + w11 * __ldg(img + o11 + 2 * C + c);
                const float d = __ldg(c1 + c) - f2;
                m11 = fmaf(gx, gx, m11); m12 = fmaf(gx, gy, m12); m22 = fmaf(gy, gy, m22); q1 = fmaf(gx, d, q1); q2 = fmaf(gy, d, q2);
            }
            m11 = warp_sum(m11); m12 = warp_sum(m12); m22 = warp_sum(m22); q1 = warp_sum(q1); q2 = warp_sum(q2);
            // ---- Jacobians (bundlenet.py:49-74) ------------------------------------------------------------------------------------
            const float a0[6] = {-fx * (x * y), -fx * (-1.f - x * x), -fx * y, -fx * (-iZ), 0.f, -fx * (x * iZ)};
            const float a1[6] = {-fy * (1.f + y * y), -fy * (-(x * y)), -fy * (-x), 0.f, -fy * (-iZ), -fy * (y * iZ)};
            const float jd0 = fx * ((rx - rz * x) * iZ), jd1 = fy * ((ry - rz * y) * iZ);
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
            // ---- 2 x (6+1) algebra (every lane, redundantly) --------------------------------------------------------------------------
            float Yc0[6], Yc1[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                float s0 = jd0 * beta[i], s1 = jd1 * beta[i];
#pragma unroll
                for (int m = 0; m < 6; ++m) { s0 = fmaf(a0[m], Scc[m * 6 + i], s0); s1 = fmaf(a1[m], Scc[m * 6 + i], s1); }
                Yc0[i] = s0; Yc1[i] = s1;
            }
            float fb0 = 0.f, fb1 = 0.f, z0 = jd0 * eta, z1 = jd1 * eta;
#pragma unroll
            for (int m = 0; m < 6; ++m) { fb0 = fmaf(a0[m], alpha[m], fb0); fb1 = fmaf(a1[m], alpha[m], fb1); z0 = fmaf(a0[m], sg[m], z0); z1 = fmaf(a1[m], sg[m], z1); }
            const float yb0 = fb0 + jd0 * gamma, yb1 = fb1 + jd1 * gamma;
            float Q00 = yb0 * jd0, Q01 = yb0 * jd1, Q10 = yb1 * jd0, Q11 = yb1 * jd1;
#pragma unroll
            for (int i = 0; i < 6; ++i) { Q00 = fmaf(Yc0[i], a0[i], Q00); Q01 = fmaf(Yc0[i], a1[i], Q01); Q10 = fmaf(Yc1[i], a0[i], Q10); Q11 = fmaf(Yc1[i], a1[i], Q11); }
            float dJ0[6], dJ1[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) { dJ0[i] = m11 * Yc0[i] + m12 * Yc1[i] + q1 * sg[i]; dJ1[i] = m12 * Yc0[i] + m22 * Yc1[i] + q2 * sg[i]; }
            const float dj0 = m11 * yb0 + m12 * yb1 + q1 * eta, dj1 = m12 * yb0 + m22 * yb1 + q2 * eta;
            const float u0 = m11 * jd0 + m12 * jd1, u1 = m12 * jd0 + m22 * jd1;
            const float sN = jd0 * u0 + jd1 * u1, tN = jd0 * q1 + jd1 * q2;
            float vN[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) vN[i] = a0[i] * u0 + a1[i] * u1;
            // ---- pass 2: dd, dG per channel -> dconv1, scatter into dconv2, coordinate gradient ------------------------------------------
            float du = 0.f, dv = 0.f;
            for (int c = lane; c < C; c += 32) {
                const float t00 = __ldg(img + o00 + c), t01 = __ldg(img + o01 + c), t10 = __ldg(img + o10 + c), t11 = __ldg(img + o11 + c);
                const float g00 = __ldg(img + o00 + C + c), g01 = __ldg(img + o01 + C + c), g10 = __ldg(img + o10 + C + c), g11 = __ldg(img + o11 + C + c);
                const float k00 = __ldg(img + o00 + 2 * C + c), k01 = __ldg(img + o01 + 2 * C + c), k10 = __ldg(img + o10 + 2 * C + c), k11 = __ldg(img + o11 + 2 * C + c);
                const float f2 = w00 * t00 + w01 * t01 + w10 * t10 + w11 * t11;
                const float gx = w00 * g00 + w01 * g01 + w10 * g10 + w11 * g11;
                const float gy = w00 * k00 + w01 * k01 + w10 * k10 + w11 * k11;
                const float d = __ldg(c1 + c) - f2;
                const float dd = gx * z0 + gy * z1 + sRh[c] * sgnf(d);
                const float dgx = gx * Q00 + gy * Q10 + d * z0, dgy = gx * Q01 + gy * Q11 + d * z1;
                dc1[c] = dd;
                const float df = -dd;
                atomicAdd(dimg + o00 + c, w00 * df); atomicAdd(dimg + o01 + c, w01 * df); atomicAdd(dimg + o10 + c, w10 * df); atomicAdd(dimg + o11 + c, w11 * df);
                atomicAdd(dimg + o00 + C + c, w00 * dgx); atomicAdd(dimg + o01 + C + c, w01 * dgx); atomicAdd(dimg + o10 + C + c, w10 * dgx); atomicAdd(dimg + o11 + C + c, w11 * dgx);
                atomicAdd(dimg + o00 + 2 * C + c, w00 * dgy); atomicAdd(dimg + o01 + 2 * C + c, w01 * dgy); atomicAdd(dimg + o10 + 2 * C + c, w10 * dgy); atomicAdd(dimg + o11 + 2 * C + c, w11 * dgy);
                du += df * ((1.f - dy) * (t01 - t00) + dy * (t11 - t10)) + dgx * ((1.f - dy) * (g01 - g00) + dy * (g11 - g10)) + dgy * ((1.f - dy) * (k01 - k00) + dy * (k11 - k10));
                dv += df * ((1.f - dx) * (t10 - t00) + dx * (t11 - t01)) + dgx * ((1.f - dx) * (g10 - g00) + dx * (g11 - g01)) + dgy * ((1.f - dx) * (k10 - k00) + dx * (k11 - k01));
            }
            du = warp_sum(du); dv = warp_sum(dv);
            // ---- geometry backward ----------------------------------------------------------------------------------------------------
            float gxx = fx * du, gyy = fy * dv, giZ = 0.f;                      // u = fx x + ox, v = fy y + oy
            gxx += -fx * (dJ0[0] * y - 2.f * x * dJ0[1] + dJ0[5] * iZ) - fy * (-dJ1[1] * y - dJ1[2]);
            gyy += -fx * (dJ0[0] * x + dJ0[2]) - fy * (2.f * y * dJ1[0] - dJ1[1] * x + dJ1[5] * iZ);
            giZ += -fx * (-dJ0[3] + dJ0[5] * x) - fy * (-dJ1[4] + dJ1[5] * y);
            float grx = dj0 * fx * iZ, gry = dj1 * fy * iZ, grz = -dj0 * fx * x * iZ - dj1 * fy * y * iZ;
            gxx += -dj0 * fx * rz * iZ; gyy += -dj1 * fy * rz * iZ;
            giZ += dj0 * fx * (rx - rz * x) + dj1 * fy * (ry - rz * y);
            const float gX = gxx * iZ, gY = gyy * iZ, gZ = -iZ * (gxx * x + gyy * y) - iZ * iZ * giZ;
            const float gDt = rx * gX + ry * gY + rz * gZ;
            grx += Dt * gX; gry += Dt * gY; grz += Dt * gZ;
            accT[0] += gX; accT[1] += gY; accT[2] += gZ;
            accR[0] += grx * p0; accR[1] += grx * p1; accR[2] += grx * p2;
            accR[3] += gry * p0; accR[4] += gry * p1; accR[5] += gry * p2;
            accR[6] += grz * p0; accR[7] += grz * p1; accR[8] += grz * p2;
            if (lane == 0) prm.dD[gi] = gDt;
            // ---- dB row, dW ---------------------------------------------------------------------------------------------------------
#pragma unroll
            for (int i = 0; i < BWD_KL; ++i) {
                const int k = lane + 32 * i;
                if (k < K) {
                    float db = sN * e[i] + tN * sg[6 + k] + gDt * sW[k];
#pragma unroll
                    for (int m = 0; m < 6; ++m) db = fmaf(vN[m], Scd[m * K + k], db);
                    prm.dB[gi * K + k] = db;
                    accW[i] = fmaf(gDt, bl[i], accW[i]);
                }
            }
        }
    }
    if (cur_b >= 0) commit(cur_b);
}

int lm_build_bwd(const banet_level_t* lv, const float* R, const float* T, const float* W, const float* dH, const float* dg, const float* drbar,
                 int exact_sym, float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW, cudaStream_t st)
{
    const int K = lv->K, P = 6 + K;
    BANET_REQUIRE(lv->conv2_channels == 3 * lv->C, BANET_ERR_UNSUPPORTED, "lm_build_bwd: conv2 must be the [F2|gx|gy] (3C) layout");
    BANET_REQUIRE(K <= 32 * BWD_KL_MAX, BANET_ERR_UNSUPPORTED, "lm_build_bwd: K=%d > %d", K, 32 * BWD_KL_MAX);
    const size_t smem = ((size_t)K * K + 12 * (size_t)K + 36 + P + K + 16 + lv->C) * sizeof(float);
    BANET_REQUIRE(smem <= 220 * 1024, BANET_ERR_UNSUPPORTED, "lm_build_bwd: K=%d, C=%d need %zu B of shared memory", K, lv->C, smem);
    void (*kern)(const BwdParams) = K <= 32 ? lm_build_bwd_kernel<1> : (K <= 128 ? lm_build_bwd_kernel<4> : lm_build_bwd_kernel<8>);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("lm_build_bwd smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    BwdParams prm;
    prm.nb = lv->nb; prm.N = lv->N; prm.C = lv->C; prm.K = K; prm.h = lv->h; prm.w = lv->w;
    prm.conv1 = lv->conv1; prm.conv2 = lv->conv2; prm.intr = lv->intr; prm.p = lv->p; prm.D = lv->D; prm.B = lv->B; prm.R = R; prm.T = T; prm.W = W;
    prm.dH = dH; prm.dg = dg; prm.drbar = drbar;
    prm.dconv1 = dconv1; prm.dconv2 = dconv2; prm.dD = dD; prm.dB = dB; prm.dR = dR; prm.dT = dT; prm.dW = dW;
    prm.exact_sym = exact_sym;
    prm.tiles_per_pair = (lv->N + BWD_TILE - 1) / BWD_TILE;
    prm.total_tiles = (long long)lv->nb * prm.tiles_per_pair;
    cudaMemsetAsync(dconv2, 0, (size_t)lv->nb * lv->h * lv->w * 3 * lv->C * sizeof(float), st);
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
// solve + update backward
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

constexpr int SB_THREADS = 1024;
__host__ __device__ __forceinline__ int tri2(int i, int k) { return i * (i + 1) / 2 + k; }

// u = Ht^-1 ddelta with the same Cholesky as lm_solve_kernel; dg (in: ddelta[0:npose] from pose_update_bwd_kernel, out: u).  npose = 6 for the
// pairs of the 2-view iteration, 6 nf for the one system of a keyframe window; the remaining P - npose entries of ddelta are dW'.
template <typename S>
__global__ void __launch_bounds__(SB_THREADS)
lm_solve_bwd_kernel(const float* __restrict__ H, const float* __restrict__ lambda, const float* __restrict__ delta, int P, int npose, float eps, int ndamped,
                    const float* __restrict__ gWn, float* __restrict__ dH, float* __restrict__ dg, float* __restrict__ dlambda, float* __restrict__ dW)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    S* A = reinterpret_cast<S*>(smraw);                 // packed lower triangle of the damped matrix -> its Cholesky factor
    S* r = A + (size_t)P * (P + 1) / 2;                 // delta (the saved forward solution)
    S* uu = r + P;                                      // ddelta -> u
    S* dgq = uu + P;                                    // sqrt of the pivots
    __shared__ int s_flag;
    __shared__ double s_dl[SB_THREADS / 32];            // per-warp partial sums of dlambda, added in a fixed order: bit-reproducible
    const int b = blockIdx.x, tid = threadIdx.x, K = P - npose;
    const float* Hb = H + (size_t)b * P * P;
    const float lam = lambda[b];
    if (tid == 0) s_flag = 0;
    __syncthreads();
    int bad = 0;
    for (int i = tid / 32; i < P; i += SB_THREADS / 32)
        for (int k = tid % 32; k <= i; k += 32) {
            const float v = Hb[(size_t)i * P + k];
            if (!isfinite(v)) bad = 1;
            S sv = (S)v;
            if (k == i && i < ndamped) sv += ((S)v + (S)eps) * (S)lam;
            A[tri2(i, k)] = sv;
        }
    for (int i = tid; i < P; i += SB_THREADS) {
        r[i] = (S)delta[(size_t)b * P + i];
        if (i < npose) uu[i] = (S)dg[(size_t)b * P + i];
        else { const float v = gWn[(size_t)b * K + i - npose]; uu[i] = (S)v; dW[(size_t)b * K + i - npose] = v; }       // W' = W + delta_d
    }
    if (!isfinite(lam)) bad = 1;
    if (bad) atomicOr(&s_flag, 2);
    const int ta = tid >> 5, tb = tid & 31;
    S inv_prev = (S)1;
    for (int j = 0; j < P; ++j) {                       // same right-looking Cholesky as lm_solve_kernel
        __syncthreads();
        if (j > 0) for (int i = j + tid; i < P; i += SB_THREADS) A[tri2(i, j - 1)] *= inv_prev;
        S d = A[tri2(j, j)];
        if (!(d > (S)0)) { if (tid == 0) atomicOr(&s_flag, 1); d = (S)1; }
        const S invd = (S)1 / d;
        inv_prev = (S)1 / sqrt(d);
        for (int i = j + 1 + ta; i < P; i += 32) {
            const S ci = A[tri2(i, j)] * invd;
            for (int k = j + 1 + tb; k <= i; k += 32) A[tri2(i, k)] -= ci * A[tri2(k, j)];
        }
        if (tid == 0) dgq[j] = sqrt(d);
    }
    __syncthreads();
    if (tid < 32) {                                     // warp 0: L y = ddelta, L^T u = y
        const int lane = tid;
        S* x = uu;
        for (int j = 0; j < P; ++j) {
            __syncwarp();
            const S yj = x[j] / dgq[j];
            __syncwarp();
            if (lane == 0) x[j] = yj;
            for (int i = j + 1 + lane; i < P; i += 32) x[i] -= A[tri2(i, j)] * yj;
        }
        for (int j = P - 1; j >= 0; --j) {
            __syncwarp();
            const S xj = x[j] / dgq[j];
            __syncwarp();
            if (lane == 0) x[j] = xj;
            for (int i = lane; i < j; i += 32) x[i] -= A[tri2(j, i)] * xj;
        }
    }
    __syncthreads();
    const int flag = s_flag;
    // dH = -u delta^T (1 + damp lambda on the diagonal), dg = u, dlambda = -sum_i u_i delta_i damp_i (H_ii + eps)
    double part = 0.0;
    for (int i = tid; i < P * P; i += SB_THREADS) {
        const int rr = i / P, cc = i - rr * P;
        float v = 0.f;
        if (!flag) {
            double t = -(double)uu[rr] * (double)r[cc];
            if (rr == cc && rr < ndamped) { part += t * ((double)Hb[(size_t)rr * P + rr] + (double)eps); t *= 1.0 + (double)lam; }
            v = (float)t;
        }
        dH[(size_t)b * P * P + i] = v;
    }
    for (int i = tid; i < P; i += SB_THREADS) dg[(size_t)b * P + i] = flag ? 0.f : (float)uu[i];
    part += __shfl_xor_sync(0xffffffffu, part, 16); part += __shfl_xor_sync(0xffffffffu, part, 8); part += __shfl_xor_sync(0xffffffffu, part, 4);
    part += __shfl_xor_sync(0xffffffffu, part, 2); part += __shfl_xor_sync(0xffffffffu, part, 1);
    if ((tid & 31) == 0) s_dl[tid >> 5] = part;
    __syncthreads();
    if (tid == 0) {
        double dl = 0.0;
        for (int wq = 0; wq < SB_THREADS / 32; ++wq) dl += s_dl[wq];
        dlambda[b] = flag ? 0.f : (float)dl;
    }
}

int launch_pose_update_bwd(const float* delta, int nb, int P, const float* R, const float* T, const float* gRn, const float* gTn,
                           float* ddelta, float* dR, float* dT, cudaStream_t st)
{
    pose_update_bwd_kernel<<<(nb + 63) / 64, 64, 0, st>>>(delta, nb, P, R, T, gRn, gTn, ddelta, dR, dT);
    BANET_CUDA_LAUNCH_CHECK("pose_update_bwd_kernel launch");
    return BANET_OK;
}

// packed lower triangle + 3 vectors in shared memory: double up to 200 KB (P <= 220), float beyond
static size_t solve_bwd_floats(int P) { return (size_t)P * (P + 1) / 2 + 3 * (size_t)P; }
static bool solve_bwd_double(int P) { return solve_bwd_floats(P) * sizeof(double) <= 200 * 1024; }
bool solve_bwd_supported(int P) { return solve_bwd_double(P) || solve_bwd_floats(P) * sizeof(float) <= 220 * 1024; }

int launch_solve_bwd(const float* H, const float* lambda, const float* delta, int nb, int P, int npose, const banet_solve_opts_t& opts,
                     const float* gWn, float* dH, float* dg, float* dlambda, float* dW, cudaStream_t st)
{
    const int ndamped = opts.undamped_last ? P - 1 : P;
    const bool use_double = solve_bwd_double(P);
    const size_t smem = solve_bwd_floats(P) * (use_double ? sizeof(double) : sizeof(float));
    BANET_REQUIRE(solve_bwd_supported(P), BANET_ERR_UNSUPPORTED, "lm_solve_bwd: P=%d does not fit shared memory", P);
    cudaError_t e;
    if (use_double) {
        e = cudaFuncSetAttribute(lm_solve_bwd_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("lm_solve_bwd smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
        lm_solve_bwd_kernel<double><<<nb, SB_THREADS, smem, st>>>(H, lambda, delta, P, npose, opts.damping_eps, ndamped, gWn, dH, dg, dlambda, dW);
    } else {
        e = cudaFuncSetAttribute(lm_solve_bwd_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("lm_solve_bwd smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
        lm_solve_bwd_kernel<float><<<nb, SB_THREADS, smem, st>>>(H, lambda, delta, P, npose, opts.damping_eps, ndamped, gWn, dH, dg, dlambda, dW);
    }
    BANET_CUDA_LAUNCH_CHECK("lm_solve_bwd_kernel launch");
    return BANET_OK;
}

int lm_solve_update_bwd(const float* H, const float* g, const float* lambda, const float* delta, int nb, int K, const banet_solve_opts_t& opts,
                        const float* R, const float* T, const float* gRn, const float* gTn, const float* gWn,
                        float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW, cudaStream_t st)
{
    (void)g;
    BANET_REQUIRE(!opts.vmatrix_batch_scramble, BANET_ERR_UNSUPPORTED,
                  "lm_solve_update_bwd: the batch-interleaved VMatrix of bundlenet.py:45 is not differentiated (use vmatrix_batch_scramble=0)");
    const int P = 6 + K;
    BANET_REQUIRE(solve_bwd_supported(P), BANET_ERR_UNSUPPORTED, "lm_solve_update_bwd: P=%d does not fit shared memory", P);
    int rc = launch_pose_update_bwd(delta, nb, P, R, T, gRn, gTn, dg, dR, dT, st);       // ddelta[0:6] parked in dg
    if (rc) return rc;
    return launch_solve_bwd(H, lambda, delta, nb, P, 6, opts, gWn, dH, dg, dlambda, dW, st);
}

}  // namespace banet
