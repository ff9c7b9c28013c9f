// lm_window.cu — joint LM step of a keyframe window: nf frame pairs (keyframe -> frame f) that share the keyframe's depth D + B.W.
//
// SURVEY.md section 8f-4.  NOT in the reference: its BA layer is 2-view (one pose + one W per pair, bundlenet.py:193-278); BA-Net's
// 5-frame use case runs it as 4 independent pairs (legacy/seq_example.py).  Here the pairs of a window share ONE W, so the unknowns are
// 6 nf + K and the normal matrix is block-arrow:
//
//        | Hcc_0              Hcd_0 |        per-pair blocks exactly as the 2-view build produces them (banet_lm_build, nb = nf):
//   Hj = |        ...          ...  |        Hcc_f 6x6, Hcd_f 6xK, Hdd_f KxK, g_f;
//        |             Hcc_nf  Hcd_nf|        the depth block and the depth right-hand side are the sums over the frames
//        | Hcd_0' ...  Hcd_nf' S Hdd |        (the residuals of all frames depend on the same W).
//
// The rest follows the 2-view iteration: lambda from the mean |residual| over ALL points of ALL frames through the same MLP
// (bundlenet.py:241-253), damping of every diagonal entry but the last depth coefficient (:264-266), one solve, every frame's pose
// updated with its own 6 entries (:269-275), W with the shared K.  The solve is the fused lm_step kernel on the one (6 nf + K) system.
//
// Training: lm_window_step with lambda given is banet_lm_window_solve_update; lm_window_step_bwd is its backward: the per-frame SE(3) update
// backward, lm_step's backward on the re-assembled system (its first 6 nf unknowns are poses), and the adjoint of the assembly.
#include "common.cuh"
#include "lm_build.h"

namespace banet {
namespace {

// C == 0: no residual statistics to sum (lambda given); zero_w == nullptr: no zero vector wanted
__global__ void window_assemble_kernel(const float* __restrict__ H, const float* __restrict__ g, const float* __restrict__ rbar_sum,
                                       int nf, int K, int C, float* __restrict__ Hj, float* __restrict__ gj, float* __restrict__ rbar_j,
                                       float* __restrict__ zero_w)
{
    const int P = 6 + K, np = 6 * nf, Pj = np + K;
    const int stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
    for (int idx = t0; idx < Pj * Pj; idx += stride) {
        const int i = idx / Pj, j = idx - i * Pj;
        float v = 0.f;
        if (i < np && j < np) {
            const int fi = i / 6, fj = j / 6;
            if (fi == fj) v = H[((size_t)fi * P + (i - 6 * fi)) * P + (j - 6 * fj)];
        } else if (i < np) {
            const int f = i / 6;
            v = H[((size_t)f * P + (i - 6 * f)) * P + 6 + (j - np)];
        } else if (j < np) {
            const int f = j / 6;
            v = H[((size_t)f * P + 6 + (i - np)) * P + (j - 6 * f)];
        } else {
            double acc = 0.0;                                       // fixed order over the frames: bit-reproducible
            for (int f = 0; f < nf; ++f) acc += (double)H[((size_t)f * P + 6 + (i - np)) * P + 6 + (j - np)];
            v = (float)acc;
        }
        Hj[idx] = v;
    }
    for (int i = t0; i < Pj; i += stride) {
        if (i < np) { const int f = i / 6; gj[i] = g[(size_t)f * P + (i - 6 * f)]; }
        else { double acc = 0.0; for (int f = 0; f < nf; ++f) acc += (double)g[(size_t)f * P + 6 + (i - np)]; gj[i] = (float)acc; }
    }
    for (int c = t0; c < C; c += stride) {
        double acc = 0.0;
        for (int f = 0; f < nf; ++f) acc += (double)rbar_sum[(size_t)f * C + c];
        rbar_j[c] = (float)acc;
    }
    if (zero_w) for (int i = t0; i < Pj; i += stride) zero_w[i] = 0.f;      // the "W" the solve kernel updates on the side (unused)
}

// Adjoint of window_assemble_kernel: every entry of a pair's (H_f, g_f) enters exactly one entry of (Hj, gj), so each thread gathers the
// gradient of its own per-pair entry (no atomics).  The depth block and the depth right-hand side are sums over the frames: every frame
// gets the whole depth-block gradient.  The cross-frame pose blocks of Hj are structural zeros and map to nothing.
__global__ void window_assemble_bwd_kernel(const float* __restrict__ dHj, const float* __restrict__ dgj, int nf, int K,
                                           float* __restrict__ dH, float* __restrict__ dg)
{
    const int P = 6 + K, np = 6 * nf, Pj = np + K;
    const int stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
    for (size_t idx = t0; idx < (size_t)nf * P * P; idx += stride) {
        const int f = (int)(idx / ((size_t)P * P)), rc = (int)(idx - (size_t)f * P * P), r = rc / P, c = rc - r * P;
        const int i = r < 6 ? 6 * f + r : np + r - 6, j = c < 6 ? 6 * f + c : np + c - 6;
        dH[idx] = dHj[(size_t)i * Pj + j];
    }
    for (int idx = t0; idx < nf * P; idx += stride) {
        const int f = idx / P, r = idx - f * P;
        dg[idx] = dgj[r < 6 ? 6 * f + r : np + r - 6];
    }
}

// W_out [w_rows,K] = W [w_rows,K] + the shared depth step (the run keeps one copy of W per frame, the single iteration one); the window's
// status goes to every frame
__global__ void window_scatter_kernel(const float* __restrict__ delta_j, const int32_t* __restrict__ status_j, int nf, int K,
                                      const float* W, int w_rows, float* W_out, int32_t* __restrict__ status, int status_accumulate)
{
    const int np = 6 * nf;
    const int stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
    for (int idx = t0; idx < w_rows * K; idx += stride) W_out[idx] = W[idx] + delta_j[np + idx % K];
    for (int f = t0; f < nf; f += stride) status[f] = status_accumulate ? (status[f] | status_j[0]) : status_j[0];
}

__global__ void window_broadcast_w_kernel(float* __restrict__ W, int nf, int K)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < (nf - 1) * K) W[K + i] = W[i % K];
}

}  // namespace

bool lm_window_supported(int nf, int K, int C) { return nf >= 1 && K >= 1 && lm_step_supported(6 * nf + K, C); }

size_t lm_window_step_workspace_floats(int nf, int K, int C)
{
    const size_t Pj = 6 * (size_t)nf + K;
    return Pj * Pj + Pj + (size_t)C + Pj + 1 + 12 + 2 * Pj + 8;
}

int lm_window_broadcast_w(float* W, int nf, int K, cudaStream_t st)
{
    if (nf > 1) {
        window_broadcast_w_kernel<<<((nf - 1) * K + 255) / 256, 256, 0, st>>>(W, nf, K);
        BANET_CUDA_LAUNCH_CHECK("window_broadcast_w_kernel launch");
    }
    return BANET_OK;
}

// One window step: assemble, the fused solve on the one (6 nf + K) system, the shared W update, the per-frame pose update.  The run calls it
// with the MLP or lambda_in, W [nf,K] in place and the status accumulated; banet_lm_window_solve_update with lambda_in (C = 0), W [1,K] and
// the caller's delta.  delta_j == nullptr: the solution goes to the workspace.
int lm_window_step(const float* H, const float* g, const float* rbar_sum, int nf, int N, int C, int K, const float* mlp, float base,
                   const float* lambda_in, const banet_solve_opts_t& opts, const float* R, const float* T, const float* W, int w_rows,
                   float* R_out, float* T_out, float* W_out, float* delta_j, float* ws, float* lambda_out, int32_t* status, int status_accumulate,
                   cudaStream_t st)
{
    const int Pj = 6 * nf + K;
    BANET_REQUIRE(lm_window_supported(nf, K, C > 0 ? C : 1), BANET_ERR_UNSUPPORTED, "lm_window_step: 6*%d+%d unknowns with C=%d do not fit the solve kernel", nf, K, C);
    float* Hj = ws;                 float* gj = Hj + (size_t)Pj * Pj;   float* rbar_j = gj + Pj;        float* delta_ws = rbar_j + C;
    float* lam = delta_ws + Pj;     float* dumR = lam + 1;
    float* dumT = dumR + 9;         float* zero_w = dumT + 3;           float* dumW = zero_w + Pj;
    int32_t* status_j = reinterpret_cast<int32_t*>(dumW + Pj);
    if (!delta_j) delta_j = delta_ws;
    window_assemble_kernel<<<64, 256, 0, st>>>(H, g, rbar_sum, nf, K, C, Hj, gj, rbar_j, zero_w);
    BANET_CUDA_LAUNCH_CHECK("window_assemble_kernel launch");
    // one system of 6 nf + K unknowns: the solve kernel sees "pose" = frame 0's six and "W" = everything else; its own pose / W outputs go
    // to scratch, the real update is the scatter below.  The mean |residual| divides by all nf * N points.
    int rc = lm_step(Hj, gj, rbar_j, 1, N * nf, C > 0 ? C : 1, Pj - 6, mlp, base, lambda_in, kStepBundleNet, nullptr, opts, R, T, zero_w, dumR, dumT, dumW,
                     delta_j, lam, status_j, 0, st);
    if (rc) return rc;
    window_scatter_kernel<<<(nf * K + 255) / 256, 256, 0, st>>>(delta_j, status_j, nf, K, W, w_rows, W_out, status, status_accumulate);
    BANET_CUDA_LAUNCH_CHECK("window_scatter_kernel launch");
    if (lambda_out) {
        cudaError_t e = cudaMemcpyAsync(lambda_out, lam, sizeof(float), cudaMemcpyDeviceToDevice, st);
        if (e != cudaSuccess) { set_error("lm_window_step: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    }
    return launch_pose_update(delta_j, nf, 6, 0, R, T, R_out, T_out, st);        // frame f's six entries are delta_j[6f, 6f+6)
}

size_t lm_window_step_bwd_workspace_floats(int nf, int K)
{
    const size_t Pj = 6 * (size_t)nf + K;
    return 2 * Pj * Pj + 2 * Pj;
}

// Backward of one window step (lambda given): with ddelta = [pose part from the per-frame SE(3) update backward | dW'], u = Ht_j^-1 ddelta
// on the re-assembled damped system gives dHj = -u delta_j^T (+ the damping terms), dgj = u and dlambda (lm_step_bwd, npose = 6 nf);
// the assembly's adjoint maps (dHj, dgj) to the pairs.  dW = dW' (W' = W + delta_d).  lm_step_bwd factors with the forward's kernel code and
// storage, and the assembled gj goes with it: a window whose forward was skipped gets zero dH, dg, dlambda.
int lm_window_step_bwd(const float* H, const float* g, const float* lambda, const float* delta_j, int nf, int K, const banet_solve_opts_t& opts,
                       const float* R, const float* T, const float* gRn, const float* gTn, const float* gWn,
                       float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW, float* ws, cudaStream_t st)
{
    const int Pj = 6 * nf + K;
    BANET_REQUIRE(lm_window_supported(nf, K, 1), BANET_ERR_UNSUPPORTED, "lm_window_step_bwd: 6*%d+%d unknowns do not fit the solve kernel", nf, K);
    float* Hj = ws; float* dHj = Hj + (size_t)Pj * Pj; float* dgj = dHj + (size_t)Pj * Pj; float* gj = dgj + Pj;
    window_assemble_kernel<<<64, 256, 0, st>>>(H, g, nullptr, nf, K, 0, Hj, gj, nullptr, nullptr);
    BANET_CUDA_LAUNCH_CHECK("window_assemble_kernel launch");
    int rc = launch_pose_update_bwd(delta_j, nf, 6, R, T, gRn, gTn, dgj, dR, dT, st);                   // ddelta[0:6 nf] -> dgj
    if (rc) return rc;
    rc = lm_step_bwd(Hj, gj, nullptr, 1, 1, 0, Pj - 6, nullptr, lambda, delta_j, opts, nullptr, nullptr, nullptr, nullptr, gWn, 6 * nf, dgj, dHj, dgj,
                     nullptr, nullptr, dlambda, nullptr, nullptr, dW, nullptr, st);
    if (rc) return rc;
    window_assemble_bwd_kernel<<<64, 256, 0, st>>>(dHj, dgj, nf, K, dH, dg);
    BANET_CUDA_LAUNCH_CHECK("window_assemble_bwd_kernel launch");
    return BANET_OK;
}

}  // namespace banet
