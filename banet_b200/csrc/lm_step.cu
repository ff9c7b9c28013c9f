// One kernel for everything of an LM iteration that is not the normal-equation build: lambda-MLP, damping, blocked Cholesky with the
// right-hand side carried as an extra row, blocked back substitution, SE(3) / depth-coefficient update.  One launch, one CTA (1024 threads)
// per pair:
//   1. rbar = rbar_sum / N, ||rbar||; 5 dense layers C->2C->4C->2C->C->1 (selu x4, tanh): warps take (32 outputs x an input slice) tasks,
//      lanes over consecutive outputs (coalesced 128-B weight rows, 8 rows in flight per lane), slices combined through shared memory;
//      lambda = base * ||rbar||^(2 + tanh(.))                                                            (bundlenet.py:243-253)
//   2. lower triangle of H (+ damping on the diagonal) and g as row P of the same array, in S = double (square to P = 157, packed to 222) or
//      float (packed, to 332), in the storage the MLP's buffers used (lm_step.cuh);
//   3. right-looking Cholesky in panels of 4 columns: one thread per row of the panel (the block's own rows, the rows below, and row P = the
//      right-hand side, so that forward substitution comes for free); every row owner factors the 4x4 diagonal block redundantly IN REGISTERS and
//      solves its own row against it (a single thread factoring through shared memory was 37 % of the first version's run time, measured);
//      warp-per-row trailing update; 3 block barriers per panel instead of one per column;
//   4. back substitution L^T x = y panel by panel (4 warps form the 4 dot products of a panel, thread 0 solves the 4x4 triangle in registers);
//   5. delta, W' = W + delta_d, status; R' = exp(w) R, T' = V(w) t + exp(w) T in double by thread 0 (per-pair VMatrix).
// The same kernel is the pair solve with lambda given (banet_lm_solve_update) and, with its backward, the dense keyframe window's solve.  The
// reference's batch-interleaved VMatrix (vmatrix_batch_scramble, bundlenet.py:45) needs every pair's delta first: the step then leaves R, T
// alone (R_out == nullptr) and pose_update_kernel follows.  banet_lm_lambda is step 1 on its own (step_lambda_kernel).
#include "lm_step.cuh"
#include "pose_bwd.cuh"

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
    auto IX = [&](int i, int k) -> int { return FULL ? i * LD + k : i * (i + 1) / 2 + k; };
    float* mbuf = reinterpret_cast<float*>(smraw);                   // MLP buffers (A's storage): 2 x 4C floats + max(4C, 1024) floats of slice partials
    S* xs = reinterpret_cast<S*>(smraw + step_vectors_offset(P, FULL, sizeof(S), lambda_in ? 0 : C));   // [P] solution
    S* dinv = xs + P;                                                // [P] reciprocals of the Cholesky diagonal
    S* dots = dinv + P;                                              // [STEP_NB]
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
        if (tid == 0 && lambda_out) lambda_out[b] = lam;
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
        if (!R_out) return;                                          // the caller updates R, T (vmatrix_batch_scramble)
        double dl[6];
        for (int i = 0; i < 6; ++i) { float dv = flag ? 0.f : (float)xs[i]; if (!isfinite(dv)) dv = 0.f; dl[i] = (double)dv; }
        se3_update(dl, mode, R + (size_t)b * 9, T + (size_t)b * 3, R_out + (size_t)b * 9, T_out + (size_t)b * 3);
    }
}

// Backward of lm_step_kernel in kStepBundleNet mode, one CTA per pair, in the forward's shared-memory layout and storage (S, FULL):
//   1. the lambda-MLP forward again with step_lambda_mlp's code, every activation kept in the pair's workspace row (nothing extra is saved by
//      the forward);
//   2. the SE(3) update backward at the forward's step (pose_bwd.cuh): ddelta[0:6], dR, dT; dW = dW';
//   3. the damped matrix factored as the forward did, with [ddelta[0:6] | dW'] as row P: u = Ht^-1 [ddelta | dW'];
//   4. dH = -u delta^T ((1 + lambda) on the damped diagonal), dg = u, dlambda (solve_adjoint_outputs);
//   5. through lambda = base ||rbar||^(2 + t), t = tanh(z_5): dt = dlambda lambda ln||rbar||, d||rbar|| = dlambda lambda (2 + t) / ||rbar||,
//      then the five layers backwards (warp per input row, fixed-order warp sums; selu' from the stored output a: scale if a > 0, else
//      a + scale alpha), each layer's output delta stored next to its input activation; drbar_sum = drbar / N.  The MLP's buffers share A's
//      storage: step 4 reads u, delta and the global H, not A.
// The skip is re-derived from H, g, lambda exactly as the forward decides it; a skipped pair gets zero dH, dg, dlambda, drbar_sum and a zero
// workspace row (no MLP contribution) and passes dR', dT', dW' through (its delta is 0).
// ddelta_pose != nullptr (the dense keyframe window, lambda given): the first npose unknowns are poses whose update backward the caller ran;
// their rows of the right-hand side come from ddelta_pose [nb, npose] (it may be dg: it is read before dg is written), step 2 is skipped and
// dR, dT are not written.  Else npose = 6.
template <typename S, bool FULL>
__global__ void __launch_bounds__(STEP_THREADS)
lm_step_bwd_kernel(const float* __restrict__ H, const float* __restrict__ g, const float* __restrict__ rbar_sum, int N, int C,
                   const float* __restrict__ mlp, const float* __restrict__ lambda, const float* __restrict__ delta, int P, int npose, float eps,
                   int ndamped, const float* __restrict__ R, const float* __restrict__ T, const float* __restrict__ gRn, const float* __restrict__ gTn,
                   const float* __restrict__ gWn, const float* ddelta_pose, float* __restrict__ dH, float* dg, float* __restrict__ drbar_sum,
                   float* __restrict__ dlambda, float* __restrict__ dR, float* __restrict__ dT, float* __restrict__ dW, float* ws)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    S* A = reinterpret_cast<S*>(smraw);                              // the forward's layout (lm_step_kernel)
    const int LD = (P + 1) | 1;
    auto IX = [&](int i, int k) -> int { return FULL ? i * LD + k : i * (i + 1) / 2 + k; };
    float* mbuf = reinterpret_cast<float*>(smraw);                   // MLP buffers as in the forward; the backward's deltas ping-pong in 2 x 4C
    S* xs = reinterpret_cast<S*>(smraw + step_vectors_offset(P, FULL, sizeof(S), mlp ? C : 0));   // [P] u
    S* dinv = xs + P;                                                // [P] reciprocals of the Cholesky diagonal, then the forward's delta
    S* dots = dinv + P;
    __shared__ int s_flag;
    __shared__ float s_wpart[STEP_WARPS], s_lam, s_lam_unused, s_ddl[6], s_dn;
    __shared__ double s_part[STEP_WARPS];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, K = P - npose;
    float* keep = mlp ? ws + (size_t)b * mlp_ws_stride(C) : nullptr;
    const float invN = 1.0f / (float)N;
    if (tid == 0) s_flag = 0;
    __syncthreads();

    // ---- 1. the forward's lambda-MLP, activations kept (lambda itself is the forward's, given) ---------------------------------------------
    if (mlp) {
        float part = 0.f;
        for (int c = tid; c < C; c += STEP_THREADS) { const float r = rbar_sum[(size_t)b * C + c] * invN; mbuf[c] = r; keep[c] = r; part += r * r; }
        step_lambda_mlp<true>(part, mbuf, C, mlp, 1.f, kStepBundleNet.lambda_exp0, s_wpart, &s_lam, &s_lam_unused, tid, keep);
    }
    const float lam = lambda[b];

    // ---- 2. SE(3) update backward at the forward's step -----------------------------------------------------------------------------------
    if (tid == 0 && !ddelta_pose) {
        double dl[6];
        for (int i = 0; i < 6; ++i) { dl[i] = delta[(size_t)b * P + i]; if (!isfinite(dl[i])) dl[i] = 0.0; }
        pose_update_bwd_one(dl, R + (size_t)b * 9, T + (size_t)b * 3, gRn + (size_t)b * 9, gTn + (size_t)b * 3, s_ddl, dR + (size_t)b * 9,
                            dT + (size_t)b * 3);
    }
    __syncthreads();

    // ---- 3. the forward's damped matrix, right-hand side [ddelta | dW'] as row P ----------------------------------------------------------
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
    for (int k = tid; k < P; k += STEP_THREADS) {
        if (!isfinite(g[(size_t)b * P + k])) bad = 1;                // the forward skipped the step on a non-finite right-hand side
        float v;
        if (k < npose) v = ddelta_pose ? ddelta_pose[(size_t)b * npose + k] : s_ddl[k];
        else { v = gWn[(size_t)b * K + k - npose]; dW[(size_t)b * K + k - npose] = v; }      // W' = W + delta_d
        A[IX(P, k)] = (S)v;
    }
    if (!isfinite(lam)) bad = 1;
    if (bad) atomicOr(&s_flag, 2);
    __syncthreads();
    step_cholesky_solve<S, FULL>(A, P, xs, dinv, dots, &s_flag, tid);

    // ---- 4. dH, dg, dlambda ----------------------------------------------------------------------------------------------------------------
    for (int i = tid; i < P; i += STEP_THREADS) dinv[i] = (S)delta[(size_t)b * P + i];
    __syncthreads();
    const int flag = s_flag;
    const float dlam = solve_adjoint_outputs<S>(xs, dinv, Hb, P, ndamped, eps, lam, flag, dH + (size_t)b * P * P, dg + (size_t)b * P, s_part, tid);
    if (tid == 0) dlambda[b] = dlam;
    if (!mlp) return;
    if (flag) {                                                      // skipped: no MLP contribution
        for (size_t i = tid; i < mlp_ws_stride(C); i += STEP_THREADS) keep[i] = 0.f;
        for (int c = tid; c < C; c += STEP_THREADS) drbar_sum[(size_t)b * C + c] = 0.f;
        return;
    }

    // ---- 5. lambda = base ||rbar||^(2 + t) and the five layers backwards (bundlenet.py:244-253) ------------------------------------------
    float* dout = mbuf; float* din = mbuf + 4 * C;
    if (tid == 0) {
        const double nrm = keep[mlp_norm_off(C)], t = keep[mlp_act_off(5, C)], L = (double)dlam * (double)lam;
        double dt = 0.0, dn = 0.0;
        if (nrm > 0.0) { dt = L * log(nrm); dn = L * (2.0 + t) / (nrm * nrm); }
        s_dn = (float)dn;                                            // drbar_i gets dn * rbar_i (d||rbar|| / d rbar_i = rbar_i / ||rbar||)
        dout[0] = (float)(dt * (1.0 - t * t));
    }
    __syncthreads();
    const float selu_scale = 1.0507009873554804934193349852946f, selu_sa = 1.0507009873554804934193349852946f * 1.6732632423543772848170429916717f;
    const int dims[6] = {C, 2 * C, 4 * C, 2 * C, C, 1};
    size_t woff[5];
    woff[0] = 0;
    for (int l = 1; l < 5; ++l) woff[l] = woff[l - 1] + (size_t)dims[l - 1] * dims[l] + dims[l];
    for (int l = 4; l >= 0; --l) {
        const int cin = dims[l], cout = dims[l + 1];
        const float* Wm = mlp + woff[l];
        for (int j = tid; j < cout; j += STEP_THREADS) keep[mlp_delta_off(l, C) + j] = dout[j];
        for (int i = warp; i < cin; i += STEP_WARPS) {                // da_i = sum_j W[i][j] delta_j: a warp per row, lanes over the row
            float s = 0.f;
            for (int j = lane; j < cout; j += 32) s = fmaf(__ldg(Wm + (size_t)i * cout + j), dout[j], s);
            s = warp_sum(s);
            if (lane == 0) {
                if (l > 0) { const float a = keep[mlp_act_off(l, C) + i]; din[i] = s * (a > 0.f ? selu_scale : a + selu_sa); }
                else drbar_sum[(size_t)b * C + i] = (s + s_dn * keep[i]) * invN;
            }
        }
        __syncthreads();
        float* tmp = dout; dout = din; din = tmp;
    }
}

// dmlp = sum over pairs, in pair order, of each layer's outer product a_{l} delta_l^T (filters) and delta_l (biases): one thread per parameter,
// no atomics (bit-reproducible, independent of what dmlp held).  Same packing as the weights: [W1, b1, ..., W5, b5].
__global__ void lm_mlp_grad_kernel(const float* __restrict__ ws, int nb, int C, float* __restrict__ dmlp)
{
    const size_t n = (size_t)20 * C * C + (size_t)10 * C + 1;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    const int dims[6] = {C, 2 * C, 4 * C, 2 * C, C, 1};
    size_t off = 0;
    int l = 0;
    for (; l < 4; ++l) {
        const size_t sz = (size_t)dims[l] * dims[l + 1] + dims[l + 1];
        if (idx < off + sz) break;
        off += sz;
    }
    const int cin = dims[l], cout = dims[l + 1];
    const size_t r = idx - off, stride = mlp_ws_stride(C);
    float s = 0.f;
    if (r < (size_t)cin * cout) {
        const int i = (int)(r / cout), j = (int)(r - (size_t)i * cout);
        const float* a = ws + mlp_act_off(l, C) + i;
        const float* d = ws + mlp_delta_off(l, C) + j;
        for (int b = 0; b < nb; ++b) s = fmaf(a[(size_t)b * stride], d[(size_t)b * stride], s);
    } else {
        const float* d = ws + mlp_delta_off(l, C) + (r - (size_t)cin * cout);
        for (int b = 0; b < nb; ++b) s += d[(size_t)b * stride];
    }
    dmlp[idx] = s;
}

// R' = exp(w) R, T' = V(w) t + exp(w) T for nb pairs from their steps delta [nb, P], thread per pair (in place is fine: a thread reads its pair
// before it writes).  scramble: V is built from the batch-interleaved skew matrices of bundlenet.py:45 (vmatrix_batch_scramble), which need
// every pair's step first.
__global__ void pose_update_kernel(const float* __restrict__ delta, int nb, int P, int scramble, const float* R, const float* T, float* R_out,
                                   float* T_out)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    double dl[6], sk[9];
    for (int i = 0; i < 6; ++i) dl[i] = delta[(size_t)b * P + i];
    if (scramble) {
        // literal bundlenet.py:45: tf.stack([...9 x [nb,1,1]...]) on axis 0, then reshape [-1,3,3]: flat[e*nb + b'] = skew entry e of pair
        // b'; matrix b takes flat[b*9 .. b*9+8]
        for (int q = 0; q < 9; ++q) {
            const int f = b * 9 + q, e = f / nb, bp = f - e * nb;
            const float* d2 = delta + (size_t)bp * P;
            const double ax = d2[0], ay = d2[1], az = d2[2];
            const double ent[9] = {0, -az, ay, az, 0, -ax, -ay, ax, 0};
            sk[q] = ent[e];
        }
    }
    const StepMode mode = kStepBundleNet;
    se3_update(dl, mode, R + (size_t)b * 9, T + (size_t)b * 3, R_out + (size_t)b * 9, T_out + (size_t)b * 3, scramble ? sk : nullptr);
}

// banet_lm_lambda: step 1 of lm_step_kernel on its own (the same code, so the same lambda bit for bit), one CTA per pair
__global__ void __launch_bounds__(STEP_THREADS)
step_lambda_kernel(const float* __restrict__ rbar_sum, int N, int C, const float* __restrict__ mlp, float base, float* __restrict__ lambda_out)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    float* mbuf = reinterpret_cast<float*>(smraw);
    __shared__ float s_wpart[STEP_WARPS], s_lam;
    const int b = blockIdx.x, tid = threadIdx.x;
    const float invN = 1.0f / (float)N;
    float part = 0.f;
    for (int c = tid; c < C; c += STEP_THREADS) { const float r = rbar_sum[(size_t)b * C + c] * invN; mbuf[c] = r; part += r * r; }
    step_lambda_mlp(part, mbuf, C, mlp, base, kStepBundleNet.lambda_exp0, s_wpart, &s_lam, lambda_out + b, tid);
}

// The storage of lm_step_kernel and of its backward, which must factor alike (the backward re-derives the forward's skip from its own
// factorisation): square double (P <= 157), packed double (P <= 222), packed float (P <= 332), from the matrix and the vectors alone.  smem
// adds the MLP's buffers where they outgrow the matrix (lm_step.cuh); Cm: the MLP width, 0 when lambda is given.
namespace {
struct StepPlan { bool full, use_double; size_t smem; };
size_t step_solve_bytes(int P, bool dbl, bool full) { return (step_matrix_elems(P, full) + 2 * (size_t)P + STEP_NB) * (dbl ? sizeof(double) : sizeof(float)); }
StepPlan step_plan(int P, int Cm)
{
    StepPlan p;
    p.full = step_solve_bytes(P, true, true) <= 200 * 1024;
    p.use_double = p.full || step_solve_bytes(P, true, false) <= 200 * 1024;
    const size_t elem = p.use_double ? sizeof(double) : sizeof(float);
    p.smem = step_vectors_offset(P, p.full, elem, Cm) + (2 * (size_t)P + STEP_NB) * elem;
    return p;
}
}  // namespace

bool lm_step_supported(int P, int Cm) { return step_plan(P, Cm).smem <= 220 * 1024; }

// lambda_in != nullptr: used as is (lambda_out, optional, receives it); else lambda = base * ||rbar||^(exp0 + MLP(rbar)) (MLP term 0 when
// mlp == nullptr).  R_out == nullptr: R, T are not updated.  In-place R/T/W (R_out == R ...) is fine: a pair's CTA reads before it writes.
int lm_step(const float* H, const float* g, const float* rbar_sum, int nb, int N, int C, int K, const float* mlp, float base, const float* lambda_in,
            const StepMode& mode, const float* nvalid, const banet_solve_opts_t& opts, const float* R, const float* T, const float* W, float* R_out, float* T_out, float* W_out,
            float* delta, float* lambda_out, int32_t* status, int status_accumulate, cudaStream_t st)
{
    const int P = 6 + K;
    const int ndamped = opts.undamped_last ? P - 1 : P;
    const StepPlan plan = step_plan(P, lambda_in ? 0 : C);
    const size_t smem = plan.smem;
    BANET_REQUIRE(smem <= 220 * 1024, BANET_ERR_UNSUPPORTED, "lm_step: P=%d, C=%d do not fit shared memory", P, C);
    auto launch = [&](auto kern) -> int {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("lm_step smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
        kern<<<nb, STEP_THREADS, smem, st>>>(H, g, rbar_sum, N, C, mlp, base, lambda_in, mode, nvalid, P, opts.damping_eps, ndamped, R, T, W,
                                             R_out, T_out, W_out, delta, lambda_out, status, status_accumulate);
        return BANET_OK;
    };
    int rc;
    if (plan.full) rc = launch(lm_step_kernel<double, true>);
    else if (plan.use_double) rc = launch(lm_step_kernel<double, false>);
    else rc = launch(lm_step_kernel<float, false>);
    if (rc) return rc;
    BANET_CUDA_LAUNCH_CHECK("lm_step_kernel launch");
    return BANET_OK;
}

int launch_pose_update(const float* delta, int nb, int P, int scramble, const float* R, const float* T, float* R_out, float* T_out, cudaStream_t st)
{
    pose_update_kernel<<<(nb + 127) / 128, 128, 0, st>>>(delta, nb, P, scramble, R, T, R_out, T_out);
    BANET_CUDA_LAUNCH_CHECK("pose_update_kernel launch");
    return BANET_OK;
}

// lm_step with lambda given; with vmatrix_batch_scramble the step leaves R, T alone and pose_update_kernel updates them from every pair's step
int lm_solve_update(const float* H, const float* g, const float* lambda, int nb, int K, const banet_solve_opts_t& opts,
                    const float* R, const float* T, const float* W, float* R_out, float* T_out, float* W_out,
                    float* delta, int32_t* status, int status_accumulate, cudaStream_t st)
{
    const bool scramble = opts.vmatrix_batch_scramble != 0;
    int rc = lm_step(H, g, nullptr, nb, 1, 0, K, nullptr, 1.f, lambda, kStepBundleNet, nullptr, opts, R, T, W, scramble ? nullptr : R_out, T_out,
                     W_out, delta, nullptr, status, status_accumulate, st);
    if (rc || !scramble) return rc;
    return launch_pose_update(delta, nb, 6 + K, 1, R, T, R_out, T_out, st);
}

int lm_lambda(const float* rbar_sum, int nb, int N, int C, const float* mlp, float base, float* lambda_out, cudaStream_t st)
{
    const size_t smem = mlp_smem_bytes(C);
    BANET_REQUIRE(smem <= 220 * 1024, BANET_ERR_UNSUPPORTED, "lm_lambda: C=%d too large", C);
    cudaError_t e = cudaFuncSetAttribute(step_lambda_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("lm_lambda smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    step_lambda_kernel<<<nb, STEP_THREADS, smem, st>>>(rbar_sum, N, C, mlp, base, lambda_out);
    BANET_CUDA_LAUNCH_CHECK("step_lambda_kernel launch");
    return BANET_OK;
}

size_t lm_step_bwd_ws_floats(int C) { return mlp_ws_stride(C); }

// Backward of lm_step (kStepBundleNet).  mlp == nullptr: lambda was given and only dlambda carries its gradient (drbar_sum, dmlp, ws unused).
// ddelta_pose != nullptr: the first npose of the P = 6 + K unknowns are poses, their update backward done by the caller (lm_step_bwd_kernel).
int lm_step_bwd(const float* H, const float* g, const float* rbar_sum, int nb, int N, int C, int K, const float* mlp, const float* lambda,
                const float* delta, const banet_solve_opts_t& opts, const float* R, const float* T, const float* gRn, const float* gTn,
                const float* gWn, int npose, const float* ddelta_pose, float* dH, float* dg, float* drbar_sum, float* dmlp, float* dlambda,
                float* dR, float* dT, float* dW, float* ws, cudaStream_t st)
{
    const int P = 6 + K;
    const int ndamped = opts.undamped_last ? P - 1 : P;
    const StepPlan plan = step_plan(P, mlp ? C : 0);
    const size_t smem = plan.smem;
    BANET_REQUIRE(smem <= 220 * 1024, BANET_ERR_UNSUPPORTED, "lm_step_bwd: P=%d, C=%d do not fit shared memory", P, C);
    auto launch = [&](auto kern) -> int {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("lm_step_bwd smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
        kern<<<nb, STEP_THREADS, smem, st>>>(H, g, rbar_sum, N, C, mlp, lambda, delta, P, npose, opts.damping_eps, ndamped, R, T, gRn, gTn, gWn,
                                             ddelta_pose, dH, dg, drbar_sum, dlambda, dR, dT, dW, ws);
        return BANET_OK;
    };
    int rc;
    if (plan.full) rc = launch(lm_step_bwd_kernel<double, true>);
    else if (plan.use_double) rc = launch(lm_step_bwd_kernel<double, false>);
    else rc = launch(lm_step_bwd_kernel<float, false>);
    if (rc) return rc;
    BANET_CUDA_LAUNCH_CHECK("lm_step_bwd_kernel launch");
    if (mlp) {
        const size_t n = (size_t)20 * C * C + (size_t)10 * C + 1;
        lm_mlp_grad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws, nb, C, dmlp);
        BANET_CUDA_LAUNCH_CHECK("lm_mlp_grad_kernel launch");
    }
    return BANET_OK;
}

// lm_step_bwd with lambda given
int lm_solve_update_bwd(const float* H, const float* g, const float* lambda, const float* delta, int nb, int K, const banet_solve_opts_t& opts,
                        const float* R, const float* T, const float* gRn, const float* gTn, const float* gWn,
                        float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW, cudaStream_t st)
{
    BANET_REQUIRE(!opts.vmatrix_batch_scramble, BANET_ERR_UNSUPPORTED,
                  "lm_solve_update_bwd: the batch-interleaved VMatrix of bundlenet.py:45 is not differentiated (use vmatrix_batch_scramble=0)");
    return lm_step_bwd(H, g, nullptr, nb, 1, 0, K, nullptr, lambda, delta, opts, R, T, gRn, gTn, gWn, 6, nullptr, dH, dg, nullptr, nullptr, dlambda,
                       dR, dT, dW, nullptr, st);
}

}  // namespace banet
