// lm_window_batch.cu — the LM step of a BATCH of keyframe windows, each solved through its block-arrow structure.
//
// A batch holds nw windows of nf frames; pair w nf + f is (keyframe of window w -> frame f) and the build (banet_lm_build on nb = nw nf pairs)
// gives its Hcc_f 6x6, Hcd_f 6xK, Hdd_f KxK, g_f.  Window w has 6 nf + K unknowns (lm_window.cu has the joint system); instead of factoring it
// dense, one CTA per window eliminates the pose blocks (Schur complement) and factors only the K x K depth system:
//
//   A. per frame, thread per frame:   Ht_cc,f = Hcc_f + lambda diag(diag Hcc_f + eps) = L_f L_f^T (6x6, double),  z_f = L_f^-1 r_f
//   B. frames in a fixed order:       Y_f = L_f^-1 Hcd_f,   S += Hdd_f - Y_f^T Y_f,   s += r_d,f - Y_f^T z_f
//      then the depth damping lambda (sum_f diag Hdd_f + eps) on every depth diagonal entry but the last (bundlenet.py:264-266)
//   C. S x_d = s: the blocked Cholesky of lm_step (lm_step.cuh) with s as the extra row
//   D. per frame, warp per frame:     x_f = Ht_cc,f^-1 (r_f - Hcd_f x_d)
//
// Only S (and one frame's Y) lives in shared memory: nothing limits nf but the workspace, which holds each frame's L_f, z_f and x_f
// (ARROW_FRAME_DOUBLES doubles).  S is double while it fits shared memory (square, then packed, as lm_step chooses for its own matrix), else float.
// No atomics: every sum over frames runs in frame order inside one thread, so the step is bit-reproducible and independent of the workspace's
// previous contents.
//
// Forward (r = g): lambda from the window's mean |residual| over its nf N points through the MLP (bundlenet.py:241-253) or given, the step,
// the per-frame SE(3) update of lm_step, W' = W + x_d.  Backward (lambda given, r = [SE(3)-update backward of dR', dT' | dW']): the same
// factorisation gives u = Ht^-1 r; dH_f, dg_f are the solve backward of lm_bwd.cu (npose = 6 nf) composed with the assembly's adjoint
// (lm_window.cu), written per pair without forming the joint matrix; dlambda is a fixed-order sum.
#include "lm_step.cuh"
#include "pose_bwd.cuh"

namespace banet {
namespace {

// per frame in the workspace: L_f (packed lower, 21), 1 / diag L_f (6), z_f (6), x_f (6), pad
constexpr int ARROW_FRAME_DOUBLES = 40;
constexpr int AF_INV = 21, AF_Z = 27, AF_X = 33;
__device__ __forceinline__ int t6(int r, int c) { return r * (r + 1) / 2 + c; }

struct ArrowParams {
    int nf, K, N, C;
    float eps, base;
    StepMode mode;                           // kStepBundleNet (bundlenet.py:241-276)
    int ndamped_d;                           // depth diagonal entries that get damping: K - 1 (the reference leaves the last undamped) or K
    const float *H, *g, *rbar_sum, *mlp, *lambda_in;
    const float *R, *T, *W;
    float *R_out, *T_out, *W_out, *W_pairs, *delta, *lambda_out;
    int32_t* status;
    int status_accumulate;
    // backward
    const float *delta_in, *gRn, *gTn, *gWn;
    float *dH, *dg, *dlambda, *dR, *dT, *dW;
    double* fws;                             // [nw, nf, ARROW_FRAME_DOUBLES]
};

// Shared memory of one window: S's lower triangle + right-hand-side row (square or packed) | x_d [K] | 1/diag [K] | dots [STEP_NB] |
// Y_f [6][K] | sum_f diag Hdd_f [K]  (all S) | lambda-MLP buffers (floats; forward with the MLP only)
size_t arrow_smem(int K, int C, bool use_double, bool full)
{
    const size_t nA = full ? (size_t)(K + 1) * ((K + 1) | 1) : (size_t)(K + 1) * (K + 2) / 2;
    const size_t mlp = C > 0 ? ((size_t)8 * C + (4 * C > 1024 ? 4 * C : 1024)) * sizeof(float) : 0;
    return (nA + 9 * (size_t)K + STEP_NB) * (use_double ? sizeof(double) : sizeof(float)) + mlp;
}

// Phases A-D above for window w with right-hand side r: pose part rhs_pose[(w nf + f) P + m] (row stride P), depth part rhs_d0 [K] (or 0)
// plus, per frame, rhs_d_frames[(w nf + f) P + 6 + k] (or nothing).  check_rhs: non-finite right-hand sides set status bit 2; bad_in != 0
// (this thread saw a non-finite input elsewhere) sets it too.  Returns the window's status (0: x_d in xs, x_f at AF_X of each frame's
// workspace slot).
template <typename S, bool FULL>
__device__ __forceinline__ int arrow_solve(const ArrowParams& p, int w, float lam, const float* rhs_pose, const float* rhs_d0, const float* rhs_d_frames,
                                           bool check_rhs, int bad_in, S* A, S* xs, S* dinv, S* dots, S* Y, S* dsum, int* s_flag, int tid)
{
    const int lane = tid & 31, warp = tid >> 5, nf = p.nf, K = p.K, P = 6 + K;
    const int LD = (K + 1) | 1;
    auto IX = [&](int i, int k) -> int { return FULL ? i * LD + k : i * (i + 1) / 2 + k; };
    double* fw = p.fws + (size_t)w * nf * ARROW_FRAME_DOUBLES;
    const float* Hw = p.H + (size_t)w * nf * P * P;

    // ---- A. per-frame 6x6 factor and z_f = L_f^-1 r_f ----------------------------------------------------------------------------------
    int bad = (isfinite(lam) && !bad_in) ? 0 : 1, notpd = 0;
    for (int f = tid; f < nf; f += STEP_THREADS) {
        const float* Hf = Hw + (size_t)f * P * P;
        const float* rf = rhs_pose + ((size_t)w * nf + f) * P;
        double* F = fw + (size_t)f * ARROW_FRAME_DOUBLES;
        double L[21], inv[6], z[6];
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
            for (int c = 0; c <= r; ++c) {
                const float v = Hf[r * P + c];
                if (!isfinite(v)) bad = 1;
                double a = (double)v;
                if (c == r) a += ((double)v + (double)p.eps) * (double)lam;          // bundlenet.py:264-266: every pose diagonal is damped
                L[t6(r, c)] = a;
            }
#pragma unroll
        for (int c = 0; c < 6; ++c) {
            double d = L[t6(c, c)];
#pragma unroll
            for (int m = 0; m < c; ++m) d -= L[t6(c, m)] * L[t6(c, m)];
            if (!(d > 0.0)) { notpd = 1; d = 1.0; }
            const double sq = sqrt(d), iv = 1.0 / sq;
            L[t6(c, c)] = sq; inv[c] = iv;
#pragma unroll
            for (int r = c + 1; r < 6; ++r) {
                double v = L[t6(r, c)];
#pragma unroll
                for (int m = 0; m < c; ++m) v -= L[t6(r, m)] * L[t6(c, m)];
                L[t6(r, c)] = v * iv;
            }
        }
#pragma unroll
        for (int m = 0; m < 6; ++m) {
            const float v = rf[m];
            if (check_rhs && !isfinite(v)) bad = 1;
            double s = (double)v;
#pragma unroll
            for (int n = 0; n < m; ++n) s -= L[t6(m, n)] * z[n];
            z[m] = s * inv[m];
        }
#pragma unroll
        for (int q = 0; q < 21; ++q) F[q] = L[q];
#pragma unroll
        for (int m = 0; m < 6; ++m) { F[AF_INV + m] = inv[m]; F[AF_Z + m] = z[m]; }
    }
    for (int i = warp; i <= K; i += STEP_WARPS) {                   // S = 0, s = r_d0 (same ownership as the accumulation below)
        const int kend = i < K ? i : K - 1;
        for (int k = lane; k <= kend; k += 32) A[IX(i, k)] = (i == K && rhs_d0) ? (S)rhs_d0[k] : (S)0;
    }
    for (int k = tid; k < K; k += STEP_THREADS) dsum[k] = (S)0;
    __syncthreads();                                                 // the frames' factors are in the workspace

    // ---- B. S = sum_f Hdd_f - Y_f^T Y_f, s = r_d - sum_f Y_f^T z_f, frames in order ----------------------------------------------------
    for (int f = 0; f < nf; ++f) {
        const float* Hf = Hw + (size_t)f * P * P;
        const double* F = fw + (size_t)f * ARROW_FRAME_DOUBLES;
        for (int j = tid; j < K; j += STEP_THREADS) {                // Y_f[:, j] = L_f^-1 Hcd_f[:, j] (Hcd_f^T row j: the lower triangle of H_f)
            double y[6];
#pragma unroll
            for (int m = 0; m < 6; ++m) {
                const float v = Hf[(size_t)(6 + j) * P + m];
                if (!isfinite(v)) bad = 1;
                double s = (double)v;
#pragma unroll
                for (int n = 0; n < m; ++n) s -= F[t6(m, n)] * y[n];
                y[m] = s * F[AF_INV + m];
                Y[m * K + j] = (S)y[m];
            }
        }
        __syncthreads();
        for (int i = warp; i <= K; i += STEP_WARPS) {
            if (i < K) {
                S yi[6];
#pragma unroll
                for (int m = 0; m < 6; ++m) yi[m] = Y[m * K + i];
                const float* hrow = Hf + (size_t)(6 + i) * P + 6;
                for (int k = lane; k <= i; k += 32) {
                    const float v = hrow[k];
                    if (!isfinite(v)) bad = 1;
                    S c = (S)v;
#pragma unroll
                    for (int m = 0; m < 6; ++m) c -= yi[m] * Y[m * K + k];
                    A[IX(i, k)] += c;
                    if (k == i) dsum[i] += (S)v;
                }
            } else {
                S zf[6];
#pragma unroll
                for (int m = 0; m < 6; ++m) zf[m] = (S)F[AF_Z + m];
                for (int k = lane; k < K; k += 32) {
                    S c = (S)0;
                    if (rhs_d_frames) {
                        const float v = rhs_d_frames[((size_t)w * nf + f) * P + 6 + k];
                        if (check_rhs && !isfinite(v)) bad = 1;
                        c = (S)v;
                    }
#pragma unroll
                    for (int m = 0; m < 6; ++m) c -= Y[m * K + k] * zf[m];
                    A[IX(K, k)] += c;
                }
            }
        }
        __syncthreads();                                             // Y is overwritten by the next frame
    }
    // depth damping on the summed diagonal (rounded to float, as the assembled joint matrix holds it), the last coefficient undamped
    for (int i = tid; i < p.ndamped_d; i += STEP_THREADS) {
        const S dv = (S)(float)dsum[i];
        A[IX(i, i)] += (dv + (S)p.eps) * (S)lam;
    }
    bad = __syncthreads_or(bad);
    notpd = __syncthreads_or(notpd);
    if (tid == 0) *s_flag = (bad ? 2 : 0) | (notpd ? 1 : 0);
    __syncthreads();

    // ---- C. S x_d = s --------------------------------------------------------------------------------------------------------------------
    step_cholesky_solve<S, FULL>(A, K, xs, dinv, dots, s_flag, tid);

    // ---- D. x_f = L_f^-T L_f^-1 (r_f - Hcd_f x_d), warp per frame -------------------------------------------------------------------------
    for (int f = warp; f < nf; f += STEP_WARPS) {
        const float* Hf = Hw + (size_t)f * P * P;
        double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int j = lane; j < K; j += 32) {
            const double xj = (double)xs[j];
#pragma unroll
            for (int m = 0; m < 6; ++m) c[m] += (double)Hf[(size_t)(6 + j) * P + m] * xj;
        }
#pragma unroll
        for (int m = 0; m < 6; ++m)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) c[m] += __shfl_xor_sync(0xffffffffu, c[m], o);
        if (lane == 0) {
            double* F = fw + (size_t)f * ARROW_FRAME_DOUBLES;
            const float* rf = rhs_pose + ((size_t)w * nf + f) * P;
            double y[6], x[6];
#pragma unroll
            for (int m = 0; m < 6; ++m) {
                double s = (double)rf[m] - c[m];
#pragma unroll
                for (int n = 0; n < m; ++n) s -= F[t6(m, n)] * y[n];
                y[m] = s * F[AF_INV + m];
            }
#pragma unroll
            for (int m = 5; m >= 0; --m) {
                double s = y[m];
#pragma unroll
                for (int n = m + 1; n < 6; ++n) s -= F[t6(n, m)] * x[n];
                x[m] = s * F[AF_INV + m];
            }
#pragma unroll
            for (int m = 0; m < 6; ++m) F[AF_X + m] = x[m];
        }
    }
    __syncthreads();
    return *s_flag;
}

template <typename S, bool FULL>
__global__ void __launch_bounds__(STEP_THREADS)
window_arrow_step_kernel(const ArrowParams p)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    const int K = p.K, nf = p.nf, Pj = 6 * nf + K;
    S* A = reinterpret_cast<S*>(smraw);
    const size_t nA = FULL ? (size_t)(K + 1) * ((K + 1) | 1) : (size_t)(K + 1) * (K + 2) / 2;
    S* xs = A + nA; S* dinv = xs + K; S* dots = dinv + K; S* Y = dots + STEP_NB; S* dsum = Y + 6 * K;
    float* mbuf = reinterpret_cast<float*>(dsum + K);
    __shared__ int s_flag;
    __shared__ float s_wpart[STEP_WARPS], s_lam;
    const int w = blockIdx.x, tid = threadIdx.x;

    // ---- lambda: the window's mean |residual| over its nf N points (the frames summed in order, as the joint assembly does) ----------------
    float lam;
    if (!p.lambda_in) {
        const float invN = 1.0f / (float)(p.N * nf);
        float part = 0.f;
        for (int c = tid; c < p.C; c += STEP_THREADS) {
            double acc = 0.0;
            for (int f = 0; f < nf; ++f) acc += (double)p.rbar_sum[((size_t)w * nf + f) * p.C + c];
            const float r = (float)acc * invN; mbuf[c] = r; part += r * r;
        }
        lam = step_lambda_mlp(part, mbuf, p.C, p.mlp, p.base, p.mode.lambda_exp0, s_wpart, &s_lam, p.lambda_out + w, tid);
    } else {
        lam = p.lambda_in[w];
        if (tid == 0 && p.lambda_out) p.lambda_out[w] = lam;
    }

    const int flag = arrow_solve<S, FULL>(p, w, lam, p.g, nullptr, p.g, true, 0, A, xs, dinv, dots, Y, dsum, &s_flag, tid);

    // ---- outputs: delta [6 nf + K] per window, W' = W + x_d (bundlenet.py:276), per-frame SE(3) update (:269-275), status ------------------
    for (int k = tid; k < K; k += STEP_THREADS) {
        float dv = flag ? 0.f : (float)xs[k];
        if (!isfinite(dv)) dv = 0.f;
        p.delta[(size_t)w * Pj + 6 * nf + k] = dv;
        const float wn = p.W[(size_t)w * K + k] + dv;
        p.W_out[(size_t)w * K + k] = wn;
        if (p.W_pairs) for (int f = 0; f < nf; ++f) p.W_pairs[((size_t)w * nf + f) * K + k] = wn;
    }
    const double* fw = p.fws + (size_t)w * nf * ARROW_FRAME_DOUBLES;
    for (int f = tid; f < nf; f += STEP_THREADS) {
        const size_t b = (size_t)w * nf + f;
        double dl[6];
        for (int m = 0; m < 6; ++m) {
            float dv = flag ? 0.f : (float)fw[(size_t)f * ARROW_FRAME_DOUBLES + AF_X + m];
            if (!isfinite(dv)) dv = 0.f;
            p.delta[(size_t)w * Pj + 6 * f + m] = dv;
            dl[m] = (double)dv;
        }
        se3_update(dl, p.mode, p.R + b * 9, p.T + b * 3, p.R_out + b * 9, p.T_out + b * 3);
        p.status[b] = p.status_accumulate ? (p.status[b] | flag) : flag;
    }
}

template <typename S, bool FULL>
__global__ void __launch_bounds__(STEP_THREADS)
window_arrow_step_bwd_kernel(const ArrowParams p)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    const int K = p.K, nf = p.nf, P = 6 + K, Pj = 6 * nf + K;
    S* A = reinterpret_cast<S*>(smraw);
    const size_t nA = FULL ? (size_t)(K + 1) * ((K + 1) | 1) : (size_t)(K + 1) * (K + 2) / 2;
    S* xs = A + nA; S* dinv = xs + K; S* dots = dinv + K; S* Y = dots + STEP_NB; S* dsum = Y + 6 * K;
    __shared__ int s_flag;
    __shared__ double s_dl[STEP_WARPS];
    const int w = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float lam = p.lambda_in[w];
    const float* dlt = p.delta_in + (size_t)w * Pj;

    // ---- per-frame SE(3) update backward: ddelta_f (parked in dg_f[0:6], the right-hand side), dR, dT; dW = dW' (W' = W + x_d) ----------
    for (int f = tid; f < nf; f += STEP_THREADS) {
        const size_t b = (size_t)w * nf + f;
        double dl[6];
        for (int m = 0; m < 6; ++m) { dl[m] = dlt[6 * f + m]; if (!isfinite(dl[m])) dl[m] = 0.0; }
        pose_update_bwd_one(dl, p.R + b * 9, p.T + b * 3, p.gRn + b * 9, p.gTn + b * 3, p.dg + b * P, p.dR + b * 9, p.dT + b * 3);
    }
    for (int k = tid; k < K; k += STEP_THREADS) p.dW[(size_t)w * K + k] = p.gWn[(size_t)w * K + k];

    // ---- u = Ht^-1 [ddelta_pose | dW'] by the forward's elimination; the forward's status is re-derived from the same inputs (H, g, lambda),
    // so a window whose step was skipped gets zero dH, dg, dlambda --------------------------------------------------------------------------
    int bad_g = 0;
    for (int i = tid; i < nf * P; i += STEP_THREADS) if (!isfinite(p.g[(size_t)w * nf * P + i])) bad_g = 1;
    const int flag = arrow_solve<S, FULL>(p, w, lam, p.dg, p.gWn + (size_t)w * K, nullptr, false, bad_g, A, xs, dinv, dots, Y, dsum, &s_flag, tid);
    const double* fw = p.fws + (size_t)w * nf * ARROW_FRAME_DOUBLES;

    // ---- dg_f = u (the depth part to every frame), dH_f = -u delta^T with (1 + lambda) on the damped diagonal, per pair ------------------
    for (int idx = tid; idx < nf * P; idx += STEP_THREADS) {
        const int f = idx / P, r = idx - f * P;
        const double u = r < 6 ? fw[(size_t)f * ARROW_FRAME_DOUBLES + AF_X + r] : (double)xs[r - 6];
        p.dg[((size_t)w * nf + f) * P + r] = flag ? 0.f : (float)u;
    }
    const size_t nH = (size_t)nf * P * P;
    float* dHw = p.dH + (size_t)w * nH;
    for (size_t idx = tid; idx < nH; idx += STEP_THREADS) {
        const int f = (int)(idx / ((size_t)P * P)), rc = (int)(idx - (size_t)f * P * P), r = rc / P, c = rc - r * P;
        float v = 0.f;
        if (!flag) {
            const double u = r < 6 ? fw[(size_t)f * ARROW_FRAME_DOUBLES + AF_X + r] : (double)xs[r - 6];
            const double d = (double)(c < 6 ? dlt[6 * f + c] : dlt[6 * nf + c - 6]);
            double t = -u * d;
            if (r == c && (r < 6 || r - 6 < p.ndamped_d)) t *= 1.0 + (double)lam;
            v = (float)t;
        }
        dHw[idx] = v;
    }
    // dlambda = sum over the damped diagonal of -u_i delta_i (Hj_ii + eps): the pose entries per frame, then the summed depth diagonal
    double part = 0.0;
    const float* Hw = p.H + (size_t)w * nH;
    for (int idx = tid; idx < 6 * nf; idx += STEP_THREADS) {
        const int f = idx / 6, m = idx - 6 * f;
        const double u = fw[(size_t)f * ARROW_FRAME_DOUBLES + AF_X + m];
        part += -u * (double)dlt[idx] * ((double)Hw[(size_t)f * P * P + m * P + m] + (double)p.eps);
    }
    for (int k = tid; k < p.ndamped_d; k += STEP_THREADS)
        part += -(double)xs[k] * (double)dlt[6 * nf + k] * ((double)(float)dsum[k] + (double)p.eps);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) s_dl[warp] = part;
    __syncthreads();
    if (tid == 0) {
        double dl = 0.0;
        for (int wq = 0; wq < STEP_WARPS; ++wq) dl += s_dl[wq];             // fixed order
        p.dlambda[w] = flag ? 0.f : (float)dl;
    }
}

// smem size and kernel variant for K unknowns of depth and C MLP channels (0: lambda given), the choice lm_step makes for its own matrix
struct ArrowPlan { bool use_double, full; size_t smem; };
ArrowPlan arrow_plan(int K, int C)
{
    ArrowPlan pl;
    pl.full = arrow_smem(K, C, true, true) <= 200 * 1024;
    pl.use_double = pl.full || arrow_smem(K, C, true, false) <= 200 * 1024;
    pl.smem = arrow_smem(K, C, pl.use_double, pl.full);
    return pl;
}

template <typename KernT>
int launch_arrow(KernT kern, int nw, size_t smem, const ArrowParams& prm, cudaStream_t st, const char* who)
{
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("%s smem attr: %s", who, cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    kern<<<nw, STEP_THREADS, smem, st>>>(prm);
    return BANET_OK;
}

}  // namespace

bool lm_window_batch_supported(int K, int C) { return K >= 1 && K <= 256 && arrow_plan(K, C).smem <= 220 * 1024; }

size_t lm_window_batch_ws_bytes(int nw, int nf) { return align_up((size_t)nw * nf * ARROW_FRAME_DOUBLES * sizeof(double), 256); }

int lm_window_batch_step(const float* H, const float* g, const float* rbar_sum, int nw, int nf, int N, int C, int K, const float* mlp, float base,
                         const float* lambda_in, const banet_solve_opts_t& opts, const float* R, const float* T, const float* W,
                         float* R_out, float* T_out, float* W_out, float* W_pairs, float* delta, float* lambda_out, int32_t* status,
                         int status_accumulate, void* ws, cudaStream_t st)
{
    const int Cm = lambda_in ? 0 : C;             // lambda_out may be null when lambda_in is given
    BANET_REQUIRE(lm_window_batch_supported(K, Cm), BANET_ERR_UNSUPPORTED, "lm_window_batch_step: K=%d, C=%d do not fit the window step", K, C);
    const ArrowPlan pl = arrow_plan(K, Cm);
    ArrowParams prm = {};
    prm.mode = kStepBundleNet;
    prm.nf = nf; prm.K = K; prm.N = N; prm.C = C; prm.eps = opts.damping_eps; prm.base = base;
    prm.ndamped_d = opts.undamped_last ? K - 1 : K;
    prm.H = H; prm.g = g; prm.rbar_sum = rbar_sum; prm.mlp = mlp; prm.lambda_in = lambda_in;
    prm.R = R; prm.T = T; prm.W = W; prm.R_out = R_out; prm.T_out = T_out; prm.W_out = W_out; prm.W_pairs = W_pairs;
    prm.delta = delta; prm.lambda_out = lambda_out; prm.status = status; prm.status_accumulate = status_accumulate;
    prm.fws = reinterpret_cast<double*>(ws);
    int rc;
    if (pl.full) rc = launch_arrow(window_arrow_step_kernel<double, true>, nw, pl.smem, prm, st, "window_arrow_step");
    else if (pl.use_double) rc = launch_arrow(window_arrow_step_kernel<double, false>, nw, pl.smem, prm, st, "window_arrow_step");
    else rc = launch_arrow(window_arrow_step_kernel<float, false>, nw, pl.smem, prm, st, "window_arrow_step");
    if (rc) return rc;
    BANET_CUDA_LAUNCH_CHECK("window_arrow_step_kernel launch");
    return BANET_OK;
}

int lm_window_batch_step_bwd(const float* H, const float* g, const float* lambda, const float* delta, int nw, int nf, int K, const banet_solve_opts_t& opts,
                             const float* R, const float* T, const float* gRn, const float* gTn, const float* gWn,
                             float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW, void* ws, cudaStream_t st)
{
    BANET_REQUIRE(lm_window_batch_supported(K, 0), BANET_ERR_UNSUPPORTED, "lm_window_batch_step_bwd: K=%d does not fit the window step", K);
    const ArrowPlan pl = arrow_plan(K, 0);
    ArrowParams prm = {};
    prm.nf = nf; prm.K = K; prm.eps = opts.damping_eps;
    prm.ndamped_d = opts.undamped_last ? K - 1 : K;
    prm.H = H; prm.g = g; prm.lambda_in = lambda; prm.R = R; prm.T = T;
    prm.delta_in = delta; prm.gRn = gRn; prm.gTn = gTn; prm.gWn = gWn;
    prm.dH = dH; prm.dg = dg; prm.dlambda = dlambda; prm.dR = dR; prm.dT = dT; prm.dW = dW;
    prm.fws = reinterpret_cast<double*>(ws);
    int rc;
    if (pl.full) rc = launch_arrow(window_arrow_step_bwd_kernel<double, true>, nw, pl.smem, prm, st, "window_arrow_step_bwd");
    else if (pl.use_double) rc = launch_arrow(window_arrow_step_bwd_kernel<double, false>, nw, pl.smem, prm, st, "window_arrow_step_bwd");
    else rc = launch_arrow(window_arrow_step_bwd_kernel<float, false>, nw, pl.smem, prm, st, "window_arrow_step_bwd");
    if (rc) return rc;
    BANET_CUDA_LAUNCH_CHECK("window_arrow_step_bwd_kernel launch");
    return BANET_OK;
}

__global__ void window_batch_broadcast_w_kernel(const float* __restrict__ W, int nw, int nf, int K, float* __restrict__ W_pairs)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < (size_t)nw * nf * K) { const size_t k = i % K, w = i / ((size_t)nf * K); W_pairs[i] = W[w * K + k]; }
}

int lm_window_batch_broadcast_w(const float* W, int nw, int nf, int K, float* W_pairs, cudaStream_t st)
{
    const size_t n = (size_t)nw * nf * K;
    window_batch_broadcast_w_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, nw, nf, K, W_pairs);
    BANET_CUDA_LAUNCH_CHECK("window_batch_broadcast_w_kernel launch");
    return BANET_OK;
}

}  // namespace banet
