// One kernel for everything of an LM iteration that is not the normal-equation build: lambda-MLP, damping, blocked Cholesky with the
// right-hand side carried as an extra row, blocked back substitution, SE(3) / depth-coefficient update.
//
// Replaces, per iteration, lm_lambda_kernel + lm_solve_kernel + pose_update_kernel (lm_solve.cu; reference bundlenet.py:241-253, 264-276):
// those are three launches of nb CTAs whose run time is pure dependent latency (measured round 1: 64 + 215..258 + 5 us, about 11 % of a cfg2
// solve).  Here: one launch, one CTA (1024 threads) per pair:
//   1. rbar = rbar_sum / N, ||rbar||; 5 dense layers C->2C->4C->2C->C->1 (selu x4, tanh): warps take (32 outputs x an input slice) tasks,
//      lanes over consecutive outputs (coalesced 128-B weight rows, 8 rows in flight per lane), slices combined through shared memory;
//      lambda = base * ||rbar||^(2 + tanh(.))                                                            (bundlenet.py:243-253)
//   2. packed lower triangle of H (+ damping on the diagonal) and g as row P of the same packed array, in S = double (P <= 200) or float;
//   3. right-looking Cholesky in panels of 4 columns: one thread per row of the panel (the block's own rows, the rows below, and row P = the
//      right-hand side, so that forward substitution comes for free); every row owner factors the 4x4 diagonal block redundantly IN REGISTERS and
//      solves its own row against it (a single thread factoring through shared memory was 37 % of the first version's run time, measured);
//      warp-per-row trailing update; 3 block barriers per panel instead of one per column;
//   4. back substitution L^T x = y panel by panel (4 warps form the 4 dot products of a panel, thread 0 solves the 4x4 triangle in registers);
//   5. delta, W' = W + delta_d, status; R' = exp(w) R, T' = V(w) t + exp(w) T in double by thread 0 (per-pair VMatrix).
// The reference's batch-interleaved VMatrix (vmatrix_batch_scramble, bundlenet.py:45) needs every pair's delta first: the host falls back to
// the three-kernel path for that option.
#include "lm_step.cuh"

namespace banet {

template <typename S, bool FULL>
__global__ void __launch_bounds__(STEP_THREADS)
lm_step_kernel(const float* __restrict__ H, const float* __restrict__ g, const float* __restrict__ rbar_sum, int N, int C,
               const float* __restrict__ mlp, float base, const float* __restrict__ lambda_in, const StepMode mode, const float* __restrict__ nvalid,
               int P, float eps, int ndamped,
               const float* __restrict__ R, const float* __restrict__ T, const float* __restrict__ W,
               float* __restrict__ R_out, float* __restrict__ T_out, float* __restrict__ W_out,
               float* __restrict__ delta, float* __restrict__ lambda_out, int32_t* __restrict__ status, int status_accumulate)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    // lower triangle of the damped matrix, rows 0..P (row P = right-hand side).  FULL: square storage with an odd row pitch (column walks over
    // consecutive rows are bank-conflict free for 64-bit words; the packed triangle's varying row offsets were 2..4-way conflicted); else packed.
    S* A = reinterpret_cast<S*>(smraw);
    const int LD = (P + 1) | 1;
    const size_t nA = FULL ? (size_t)(P + 1) * LD : (size_t)(P + 1) * (P + 2) / 2;
    auto IX = [&](int i, int k) -> int { return FULL ? i * LD + k : i * (i + 1) / 2 + k; };
    S* xs = A + nA;                                                  // [P] solution
    S* dinv = xs + P;                                                // [P] reciprocals of the Cholesky diagonal
    S* dots = dinv + P;                                              // [STEP_NB]
    float* mbuf = reinterpret_cast<float*>(dots + STEP_NB);          // MLP buffers: 2 x 4C floats + max(4C, 1024) floats of slice partials
    __shared__ int s_flag;
    __shared__ float s_wpart[STEP_WARPS], s_lam;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, K = P - 6;
    if (tid == 0) s_flag = 0;
    __syncthreads();

    // ---- 1. lambda -------------------------------------------------------------------------------------------------------------------
    float lam;
    if (!lambda_in) {
        // bundlenet.py:243 divides by N; the legacy tracker rescales by N / valid, i.e. divides by the in-bounds count (legacy/ba.py:256,274)
        const float invN = 1.0f / (mode.rbar_per_valid ? nvalid[b] : (float)N);
        float part = 0.f;
        for (int c = tid; c < C; c += STEP_THREADS) { const float r = rbar_sum[(size_t)b * C + c] * invN; mbuf[c] = r; part += r * r; }
        lam = step_lambda_mlp(part, mbuf, C, mlp, base, mode.lambda_exp0, s_wpart, &s_lam, lambda_out + b, tid);
    } else {
        lam = lambda_in[b];
        if (tid == 0) lambda_out[b] = lam;
    }

    // ---- 2. load (+ damping, bundlenet.py:264-266 / :181-182) -------------------------------------------------------------------------------
    const float* Hb = H + (size_t)b * P * P;
    int bad = 0;
    for (int i = warp; i < P; i += STEP_WARPS)
        for (int k = lane; k <= i; k += 32) {
            const float v = Hb[(size_t)i * P + k];
            if (!isfinite(v)) bad = 1;
            S sv = (S)v;
            if (k == i && i < ndamped) sv += ((S)v + (S)eps) * (S)lam;
            A[IX(i, k)] = sv;
        }
    for (int k = tid; k < P; k += STEP_THREADS) { const float v = g[(size_t)b * P + k]; if (!isfinite(v)) bad = 1; A[IX(P, k)] = (S)v; }
    if (!isfinite(lam)) bad = 1;
    if (bad) atomicOr(&s_flag, 2);
    __syncthreads();

    // ---- 3./4. blocked Cholesky (row P rides along: afterwards A[P][:] = y = L^-1 g) and back substitution (lm_step.cuh) ----------------------
    step_cholesky_solve<S, FULL>(A, P, xs, dinv, dots, &s_flag, tid);

    // ---- 5. outputs ----------------------------------------------------------------------------------------------------------------------------
    const int flag = s_flag;
    for (int i = tid; i < P; i += STEP_THREADS) {
        float dv = flag ? 0.f : (float)xs[i];
        if (!isfinite(dv)) dv = 0.f;
        delta[(size_t)b * P + i] = dv;
        if (i >= 6) W_out[(size_t)b * K + i - 6] = W[(size_t)b * K + i - 6] + dv;      // bundlenet.py:276
    }
    if (tid == 0) {
        status[b] = status_accumulate ? (status[b] | flag) : flag;
        double dl[6];
        for (int i = 0; i < 6; ++i) { float dv = flag ? 0.f : (float)xs[i]; if (!isfinite(dv)) dv = 0.f; dl[i] = (double)dv; }
        se3_update(dl, mode, R + (size_t)b * 9, T + (size_t)b * 3, R_out + (size_t)b * 9, T_out + (size_t)b * 3);
    }
}

size_t lm_step_smem(int P, int C, bool use_double, bool full)
{
    const size_t nA = (full ? (size_t)(P + 1) * ((P + 1) | 1) : (size_t)(P + 1) * (P + 2) / 2) + 2 * (size_t)P + STEP_NB;
    return nA * (use_double ? sizeof(double) : sizeof(float)) + ((size_t)8 * C + (4 * C > 1024 ? 4 * C : 1024)) * sizeof(float);
}

bool lm_step_supported(int P, int C) { return lm_step_smem(P, C, false, false) <= 220 * 1024; }

// lambda_in != nullptr: used as is; else lambda = base * ||rbar||^(exp0 + MLP(rbar)) (MLP term 0 when mlp == nullptr).
// In-place R/T/W (R_out == R ...) is fine: a pair's CTA reads before it writes.
int lm_step(const float* H, const float* g, const float* rbar_sum, int nb, int N, int C, int K, const float* mlp, float base, const float* lambda_in,
            const StepMode& mode, const float* nvalid, const banet_solve_opts_t& opts, const float* R, const float* T, const float* W, float* R_out, float* T_out, float* W_out,
            float* delta, float* lambda_out, int32_t* status, int status_accumulate, cudaStream_t st)
{
    const int P = 6 + K;
    const int ndamped = opts.undamped_last ? P - 1 : P;
    // storage: square double (P <= ~150), packed double (P <= ~200), packed float beyond
    const bool full = lm_step_smem(P, C, true, true) <= 200 * 1024;
    const bool use_double = full || lm_step_smem(P, C, true, false) <= 200 * 1024;
    const size_t smem = lm_step_smem(P, C, use_double, full);
    BANET_REQUIRE(smem <= 220 * 1024, BANET_ERR_UNSUPPORTED, "lm_step: P=%d, C=%d do not fit shared memory", P, C);
    auto launch = [&](auto kern) -> int {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("lm_step smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
        kern<<<nb, STEP_THREADS, smem, st>>>(H, g, rbar_sum, N, C, mlp, base, lambda_in, mode, nvalid, P, opts.damping_eps, ndamped, R, T, W,
                                             R_out, T_out, W_out, delta, lambda_out, status, status_accumulate);
        return BANET_OK;
    };
    int rc;
    if (full) rc = launch(lm_step_kernel<double, true>);
    else if (use_double) rc = launch(lm_step_kernel<double, false>);
    else rc = launch(lm_step_kernel<float, false>);
    if (rc) return rc;
    BANET_CUDA_LAUNCH_CHECK("lm_step_kernel launch");
    return BANET_OK;
}

}  // namespace banet
