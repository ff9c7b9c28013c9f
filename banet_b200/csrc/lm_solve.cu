// Damping prediction, damped normal-equation solve and SE(3)/depth update of one LM iteration.
//
// Replaces reference bundlenet.py:241-253 (lambda MLP), :264-267 (damping + tf.matrix_solve) and
// :269-276 (AngleaAxisRotation :17-37, VMatrix :39-46, pose/depth update); pose-only twin :165-190.
#include "common.cuh"
#include "lm_build.h"

namespace banet {

// ------------------------------------------------------------------------------------------------
// lambda MLP: one CTA per pair.  5 dense layers (conv1d with kernel width 1, bundlenet.py:102-110).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float selu_f(float x) {
    const float alpha = 1.6732632423543772848170429916717f, scale = 1.0507009873554804934193349852946f;
    return scale * (x > 0.f ? x : alpha * expm1f(x));
}

__global__ void __launch_bounds__(1024)
lm_lambda_kernel(const float* __restrict__ rbar_sum, int N, int C, const float* __restrict__ mlp, float base,
                 float* __restrict__ lambda_out)
{
    extern __shared__ float sm[];
    float* bufA = sm;               // up to 4C
    float* bufB = sm + 4 * C;       // up to 4C
    __shared__ float s_norm2, s_wpart[32];
    const int b = blockIdx.x, tid = threadIdx.x;
    const float invN = 1.0f / (float)N;
    float part = 0.f;
    for (int c = tid; c < C; c += blockDim.x) {
        const float r = rbar_sum[(size_t)b * C + c] * invN;           // tf.reduce_mean over N (bundlenet.py:243)
        bufA[c] = r; part += r * r;
    }
    part = warp_sum(part);
    if ((tid & 31) == 0) s_wpart[tid >> 5] = part;
    __syncthreads();
    if (tid == 0) {                                                     // fixed order: bit-reproducible (a float atomic here was not)
        float t = 0.f;
        for (int wq = 0; wq < (int)((blockDim.x + 31) >> 5); ++wq) t += s_wpart[wq];
        s_norm2 = t;
    }
    __syncthreads();
    const int dims[6] = {C, 2 * C, 4 * C, 2 * C, C, 1};
    const float* wp = mlp;
    float* in = bufA; float* out = bufB;
    for (int l = 0; l < 5; ++l) {
        const int cin = dims[l], cout = dims[l + 1];
        const float* Wm = wp; const float* bias = wp + (size_t)cin * cout;
        // 8 consecutive lanes share one output neuron j and split the input dimension; lanes of a warp that hold the
        // same input index read 4 consecutive weights (coalesced 16-B segments), partial sums meet through shuffles
        for (int j0 = 0; j0 < cout; j0 += blockDim.x / 8) {
            const int j = j0 + (tid >> 3), part = tid & 7;
            float a0 = 0.f, a1 = 0.f;
            if (j < cout) {
                int i = part;
                for (; i + 8 < cin; i += 16) {
                    a0 = fmaf(in[i], __ldg(Wm + (size_t)i * cout + j), a0);
                    a1 = fmaf(in[i + 8], __ldg(Wm + (size_t)(i + 8) * cout + j), a1);
                }
                for (; i < cin; i += 8) a0 = fmaf(in[i], __ldg(Wm + (size_t)i * cout + j), a0);
            }
            float z = a0 + a1;
            z += __shfl_xor_sync(0xffffffffu, z, 4); z += __shfl_xor_sync(0xffffffffu, z, 2); z += __shfl_xor_sync(0xffffffffu, z, 1);
            if (j < cout && part == 0) { z += __ldg(bias + j); out[j] = (l == 4) ? tanhf(z) : selu_f(z); }
        }
        __syncthreads();
        wp = bias + cout;
        float* tmp = in; in = out; out = tmp;
    }
    if (tid == 0) {
        const float nrm = sqrtf(s_norm2);
        lambda_out[b] = base * powf(nrm, 2.0f + in[0]);               // bundlenet.py:249,253
    }
}

int lm_lambda(const float* rbar_sum, int nb, int N, int C, const float* mlp, float base, float* lambda_out, cudaStream_t st)
{
    const size_t smem = (size_t)8 * C * sizeof(float);
    BANET_REQUIRE(smem <= 160 * 1024, BANET_ERR_UNSUPPORTED, "lm_lambda: C=%d too large", C);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(lm_lambda_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("lm_lambda smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    }
    lm_lambda_kernel<<<nb, 1024, smem, st>>>(rbar_sum, N, C, mlp, base, lambda_out);
    BANET_CUDA_LAUNCH_CHECK("lm_lambda_kernel launch");
    return BANET_OK;
}

// ------------------------------------------------------------------------------------------------
// Damped solve: one CTA per pair, packed lower-triangular Cholesky in shared memory.
// S = double when the packed matrix fits (P <= 223), float beyond.
// ------------------------------------------------------------------------------------------------
constexpr int SOLVE_THREADS = 1024;
__host__ __device__ __forceinline__ int tri(int i, int k) { return i * (i + 1) / 2 + k; }

template <typename S>
__global__ void __launch_bounds__(SOLVE_THREADS)
lm_solve_kernel(const float* __restrict__ H, const float* __restrict__ g, const float* __restrict__ lambda,
                int P, float eps, int ndamped, const float* __restrict__ W, float* __restrict__ W_out,
                float* __restrict__ delta, int32_t* __restrict__ status, int status_accumulate)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    S* A = reinterpret_cast<S*>(smraw);                 // packed lower triangle, P(P+1)/2
    S* r = A + (size_t)P * (P + 1) / 2;                 // rhs / solution, P
    S* dg = r + P;                                      // sqrt of the pivots, P
    __shared__ int s_flag;
    const int b = blockIdx.x, tid = threadIdx.x;
    const float* Hb = H + (size_t)b * P * P;
    const float lam = lambda[b];
    if (tid == 0) s_flag = 0;
    __syncthreads();

    // load lower triangle (+ damping on the diagonal, bundlenet.py:264-266 / :181-182)
    int bad = 0;
    for (int i = tid / 32; i < P; i += SOLVE_THREADS / 32) {
        for (int k = tid % 32; k <= i; k += 32) {
            float v = Hb[(size_t)i * P + k];
            if (!isfinite(v)) bad = 1;
            S sv = (S)v;
            if (k == i && i < ndamped) sv += ((S)v + (S)eps) * (S)lam;
            A[tri(i, k)] = sv;
        }
    }
    for (int i = tid; i < P; i += SOLVE_THREADS) {
        const float v = g[(size_t)b * P + i];
        if (!isfinite(v)) bad = 1;
        r[i] = (S)v;
    }
    if (!isfinite(lam)) bad = 1;
    if (bad) atomicOr(&s_flag, 2);

    // right-looking Cholesky; column j is scaled one iteration late (saves a barrier per column)
    const int ta = tid >> 5, tb = tid & 31;
    S inv_prev = (S)1;
    for (int j = 0; j < P; ++j) {
        __syncthreads();
        if (j > 0) {                                     // finish column j-1: L[i][j-1] = A[i][j-1]/sqrt(d)
            for (int i = j + tid; i < P; i += SOLVE_THREADS) A[tri(i, j - 1)] *= inv_prev;
        }
        S d = A[tri(j, j)];
        if (!(d > (S)0)) { if (tid == 0) atomicOr(&s_flag, 1); d = (S)1; }
        const S invd = (S)1 / d;
        inv_prev = (S)1 / sqrt(d);
        for (int i = j + 1 + ta; i < P; i += 32) {
            const S ci = A[tri(i, j)] * invd;
            for (int k = j + 1 + tb; k <= i; k += 32) A[tri(i, k)] -= ci * A[tri(k, j)];
        }
        if (tid == 0) dg[j] = sqrt(d);
    }
    __syncthreads();
    // (the last column has no sub-diagonal entries to scale)

    // substitutions on warp 0: L y = g, then L^T x = y
    if (tid < 32) {
        const int lane = tid;
        for (int j = 0; j < P; ++j) {
            __syncwarp();
            const S yj = r[j] / dg[j];
            __syncwarp();
            if (lane == 0) r[j] = yj;
            for (int i = j + 1 + lane; i < P; i += 32) r[i] -= A[tri(i, j)] * yj;
        }
        for (int j = P - 1; j >= 0; --j) {
            __syncwarp();
            const S xj = r[j] / dg[j];
            __syncwarp();
            if (lane == 0) r[j] = xj;
            for (int i = lane; i < j; i += 32) r[i] -= A[tri(j, i)] * xj;
        }
    }
    __syncthreads();
    const int flag = s_flag;
    const int K = P - 6;
    for (int i = tid; i < P; i += SOLVE_THREADS) {
        float dv = flag ? 0.f : (float)r[i];
        if (!isfinite(dv)) dv = 0.f;
        delta[(size_t)b * P + i] = dv;
        if (i >= 6) W_out[(size_t)b * K + i - 6] = W[(size_t)b * K + i - 6] + dv;      // bundlenet.py:276
    }
    if (tid == 0) status[b] = status_accumulate ? (status[b] | flag) : flag;
}

// ------------------------------------------------------------------------------------------------
// Pose update: thread per pair (bundlenet.py:269-275).  Double precision on the 3x3 algebra.
// ------------------------------------------------------------------------------------------------
__global__ void pose_update_kernel(const float* __restrict__ delta, int nb, int P, int scramble,
                                   const float* __restrict__ R, const float* __restrict__ T,
                                   float* __restrict__ R_out, float* __restrict__ T_out)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const float* dl = delta + (size_t)b * P;
    const double wx = dl[0], wy = dl[1], wz = dl[2], tx = dl[3], ty = dl[4], tz = dl[5];
    const double th_raw = sqrt(wx * wx + wy * wy + wz * wz);
    // AngleaAxisRotation (bundlenet.py:17-37): theta clamped to >= 1e-6, axis = w / theta
    const double th = fmax(th_raw, 1e-6);
    const double kx = wx / th, ky = wy / th, kz = wz / th, c = cos(th), s = sin(th), oc = 1.0 - c;
    const double dr[9] = {c + kx * kx * oc,      kx * ky * oc - kz * s, ky * s + kx * kz * oc,
                          kz * s + kx * ky * oc, c + ky * ky * oc,      -kx * s + ky * kz * oc,
                          -ky * s + kx * kz * oc, kx * s + ky * kz * oc, c + kz * kz * oc};
    // VMatrix (bundlenet.py:39-46): unclamped theta in the reference (0/0 at w = 0); series below 1e-4
    double ca, cb;
    if (th_raw < 1e-4) { ca = 0.5 - th_raw * th_raw / 24.0; cb = 1.0 / 6.0 - th_raw * th_raw / 120.0; }
    else { ca = (1.0 - cos(th_raw)) / (th_raw * th_raw); cb = (th_raw - sin(th_raw)) / (th_raw * th_raw * th_raw); }
    double sk[9];
    if (!scramble) {
        sk[0] = 0; sk[1] = -wz; sk[2] = wy; sk[3] = wz; sk[4] = 0; sk[5] = -wx; sk[6] = -wy; sk[7] = wx; sk[8] = 0;
    } else {
        // literal bundlenet.py:45: tf.stack([...9 x [nb,1,1]...]) on axis 0, then reshape [-1,3,3]:
        // flat[e*nb + b'] = skew entry e of pair b';  matrix b takes flat[b*9 .. b*9+8]
        for (int q = 0; q < 9; ++q) {
            const int f = b * 9 + q, e = f / nb, bp = f - e * nb;
            const float* d2 = delta + (size_t)bp * P;
            const double ax = d2[0], ay = d2[1], az = d2[2];
            const double ent[9] = {0, -az, ay, az, 0, -ax, -ay, ax, 0};
            sk[q] = ent[e];
        }
    }
    double sk2[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j)
        sk2[i * 3 + j] = sk[i * 3] * sk[j] + sk[i * 3 + 1] * sk[3 + j] + sk[i * 3 + 2] * sk[6 + j];
    double V[9];
    for (int q = 0; q < 9; ++q) V[q] = ((q % 4 == 0) ? 1.0 : 0.0) + ca * sk[q] + cb * sk2[q];
    double Rin[9], Tin[3];
    for (int q = 0; q < 9; ++q) Rin[q] = R[(size_t)b * 9 + q];
    for (int q = 0; q < 3; ++q) Tin[q] = T[(size_t)b * 3 + q];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j)
            R_out[(size_t)b * 9 + i * 3 + j] = (float)(dr[i * 3] * Rin[j] + dr[i * 3 + 1] * Rin[3 + j] + dr[i * 3 + 2] * Rin[6 + j]);
        T_out[(size_t)b * 3 + i] = (float)(V[i * 3] * tx + V[i * 3 + 1] * ty + V[i * 3 + 2] * tz
                                           + dr[i * 3] * Tin[0] + dr[i * 3 + 1] * Tin[1] + dr[i * 3 + 2] * Tin[2]);
    }
}

int launch_pose_update(const float* delta, int nb, int P, const float* R, const float* T, float* R_out, float* T_out, cudaStream_t st)
{
    pose_update_kernel<<<(nb + 127) / 128, 128, 0, st>>>(delta, nb, P, 0, R, T, R_out, T_out);     // every thread reads its pair before it writes: in place is fine
    BANET_CUDA_LAUNCH_CHECK("pose_update_kernel launch");
    return BANET_OK;
}

// lm_solve_kernel<double> while its packed triangle fits 200 KB (P <= 223); its backward (lm_bwd.cu) factors in the same precision
bool lm_solve_uses_double(int P) { return ((size_t)P * (P + 1) / 2 + 2 * (size_t)P) * sizeof(double) <= 200 * 1024; }

int lm_solve_update(const float* H, const float* g, const float* lambda, int nb, int K, const banet_solve_opts_t& opts,
                    const float* R, const float* T, const float* W, float* R_out, float* T_out, float* W_out,
                    float* delta, int32_t* status, int status_accumulate, cudaStream_t st)
{
    const int P = 6 + K;
    const int ndamped = opts.undamped_last ? P - 1 : P;
    const size_t ntri = (size_t)P * (P + 1) / 2 + 2 * (size_t)P;
    const bool use_double = lm_solve_uses_double(P);
    const size_t smem = ntri * (use_double ? sizeof(double) : sizeof(float));
    BANET_REQUIRE(smem <= 220 * 1024, BANET_ERR_UNSUPPORTED, "lm_solve: P=%d does not fit shared memory", P);
    cudaError_t e;
    if (use_double) {
        e = cudaFuncSetAttribute(lm_solve_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("lm_solve smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
        lm_solve_kernel<double><<<nb, SOLVE_THREADS, smem, st>>>(H, g, lambda, P, opts.damping_eps, ndamped, W, W_out, delta, status, status_accumulate);
    } else {
        e = cudaFuncSetAttribute(lm_solve_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("lm_solve smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
        lm_solve_kernel<float><<<nb, SOLVE_THREADS, smem, st>>>(H, g, lambda, P, opts.damping_eps, ndamped, W, W_out, delta, status, status_accumulate);
    }
    BANET_CUDA_LAUNCH_CHECK("lm_solve_kernel launch");
    pose_update_kernel<<<(nb + 127) / 128, 128, 0, st>>>(delta, nb, P, opts.vmatrix_batch_scramble, R, T, R_out, T_out);
    BANET_CUDA_LAUNCH_CHECK("pose_update_kernel launch");
    return BANET_OK;
}

}  // namespace banet
