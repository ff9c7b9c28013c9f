// Device code of the fused LM step shared by lm_step.cu (one CTA per pair) and lm_window_batch.cu (one CTA per keyframe window):
// the lambda-MLP, the blocked Cholesky with the right-hand side carried as an extra row, and the per-pair SE(3) update.  Every function is
// force-inlined into the kernel that calls it: moving them here left lm_step_kernel's floating-point instructions as they were (same count
// of every kind; only register allocation and scheduling moved) and its outputs bit for bit the same.
#pragma once
#include "common.cuh"
#include "lm_build.h"

namespace banet {

constexpr int STEP_THREADS = 1024;
constexpr int STEP_WARPS = STEP_THREADS / 32;
constexpr int STEP_NB = 4;                       // Cholesky panel width (the panel owners keep the NB x NB block in registers: 1024 threads leave 64 registers each)

// Dynamic shared memory of a damped step (lm_step_kernel, lm_step_bwd_kernel, the arrow's kernels): [ union(A, MLP buffers) | vectors ].
// A is the matrix of n unknowns with the right-hand side as row n (square with row pitch (n + 1) | 1, or packed), at offset 0.  The
// lambda-MLP's buffers (step_lambda_mlp) share A's storage: the MLP finishes, with a block barrier, before A is loaded, and the step's
// backward reuses them only after the factor is dead.  So the storage variant depends on the matrix and the vectors alone, and the MLP width
// Cm (0 when lambda is given) only on whether the whole fits.
__host__ __device__ __forceinline__ size_t mlp_smem_bytes(int Cm) { return Cm > 0 ? ((size_t)8 * Cm + (4 * Cm > 1024 ? 4 * Cm : 1024)) * sizeof(float) : 0; }
__host__ __device__ __forceinline__ size_t step_matrix_elems(int n, bool full) { return full ? (size_t)(n + 1) * ((n + 1) | 1) : (size_t)(n + 1) * (n + 2) / 2; }
__host__ __device__ __forceinline__ size_t step_vectors_offset(int n, bool full, size_t elem, int Cm)
{
    const size_t a = step_matrix_elems(n, full) * elem, m = mlp_smem_bytes(Cm);
    return a > m ? a : m;
}

__device__ __forceinline__ float selu_s(float x) {
    const float alpha = 1.6732632423543772848170429916717f, scale = 1.0507009873554804934193349852946f;
    return scale * (x > 0.f ? x : alpha * expm1f(x));
}

// one dense layer: out[j] = act(bias[j] + sum_i in[i] W[i][j]);  W row-major [cin][cout].  Tasks = (32-output block) x (input slice); every task
// stores its partial sums into its own row of `part` ([slices][cout], at most max(1024, cout) floats) and the activation pass adds the slices in
// a fixed order: bit-reproducible (shared-memory float atomics were not: lambda, and with it the whole step, moved in the last ulp run to run).
__device__ __forceinline__ void dense_layer(const float* __restrict__ in, const float* __restrict__ Wm, const float* __restrict__ bias,
                                            int cin, int cout, bool last, float* __restrict__ part, float* __restrict__ out, int tid)
{
    const int lane = tid & 31, warp = tid >> 5;
    const int jblocks = (cout + 31) / 32;
    int slices = STEP_WARPS / jblocks; if (slices < 1) slices = 1; if (slices > cin / 8) slices = max(1, cin / 8);
    const int ntask = jblocks * slices;
    const int rows = (cin + slices - 1) / slices;
    for (int t = warp; t < ntask; t += STEP_WARPS) {
        const int jb = t % jblocks, sl = t / jblocks;
        const int j = jb * 32 + lane, i0 = sl * rows, i1 = min(cin, i0 + rows);
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        if (j < cout) {
            int i = i0;
            for (; i + 15 < i1; i += 16) {                       // 16 weight rows in flight per lane (the loop is pure L2 latency)
                float wv[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) wv[u] = __ldg(Wm + (size_t)(i + u) * cout + j);
#pragma unroll
                for (int u = 0; u < 16; u += 4) {
                    a0 = fmaf(in[i + u], wv[u], a0); a1 = fmaf(in[i + u + 1], wv[u + 1], a1); a2 = fmaf(in[i + u + 2], wv[u + 2], a2); a3 = fmaf(in[i + u + 3], wv[u + 3], a3);
                }
            }
            for (; i + 7 < i1; i += 8) {
                const float w0 = __ldg(Wm + (size_t)i * cout + j), w1 = __ldg(Wm + (size_t)(i + 1) * cout + j), w2 = __ldg(Wm + (size_t)(i + 2) * cout + j),
                            w3 = __ldg(Wm + (size_t)(i + 3) * cout + j), w4 = __ldg(Wm + (size_t)(i + 4) * cout + j), w5 = __ldg(Wm + (size_t)(i + 5) * cout + j),
                            w6 = __ldg(Wm + (size_t)(i + 6) * cout + j), w7 = __ldg(Wm + (size_t)(i + 7) * cout + j);
                a0 = fmaf(in[i], w0, a0); a1 = fmaf(in[i + 1], w1, a1); a2 = fmaf(in[i + 2], w2, a2); a3 = fmaf(in[i + 3], w3, a3);
                a0 = fmaf(in[i + 4], w4, a0); a1 = fmaf(in[i + 5], w5, a1); a2 = fmaf(in[i + 6], w6, a2); a3 = fmaf(in[i + 7], w7, a3);
            }
            for (; i < i1; ++i) a0 = fmaf(in[i], __ldg(Wm + (size_t)i * cout + j), a0);
            part[sl * cout + j] = (a0 + a1) + (a2 + a3);
        }
    }
    __syncthreads();
    for (int j = tid; j < cout; j += STEP_THREADS) {
        float z = part[j];
        for (int sl = 1; sl < slices; ++sl) z += part[sl * cout + j];
        z += __ldg(bias + j);
        out[j] = last ? tanhf(z) : selu_s(z);
    }
    __syncthreads();
}

// lambda = base * ||rbar||^(exp0 + MLP(rbar)) (bundlenet.py:243-253; MLP term 0 when mlp == nullptr).  On entry mbuf[0:C] holds rbar and `part`
// is this thread's share of ||rbar||^2; mbuf: 2 x 4C floats + max(4C, 1024) floats of slice partials.  Thread 0 writes *lambda_out.
// KEEP (the step's backward): the same arithmetic, and layer l's output activation also goes to keep + mlp_act_off(l + 1, C) and ||rbar||
// to keep[mlp_norm_off(C)].  That is the per-pair workspace row of lm_step_bwd: activations a_0 = rbar (stored by the caller), a_1..a_5,
// then each layer's output delta (the gradient of its pre-activation), then ||rbar||.
__host__ __device__ __forceinline__ int mlp_act_off(int l, int C) { const int o[6] = {0, C, 3 * C, 7 * C, 9 * C, 10 * C}; return o[l]; }
__host__ __device__ __forceinline__ int mlp_delta_off(int l, int C) { const int o[5] = {10 * C + 1, 12 * C + 1, 16 * C + 1, 18 * C + 1, 19 * C + 1}; return o[l]; }
__host__ __device__ __forceinline__ int mlp_norm_off(int C) { return 19 * C + 2; }
__host__ __device__ __forceinline__ size_t mlp_ws_stride(int C) { return ((size_t)19 * C + 3 + 3) & ~(size_t)3; }   // floats per pair, 16-B rows

template <bool KEEP = false>
__device__ __forceinline__ float step_lambda_mlp(float part, float* mbuf, int C, const float* __restrict__ mlp, float base, float exp0,
                                                 float* s_wpart, float* s_lam, float* lambda_out, int tid, float* keep = nullptr)
{
    const int lane = tid & 31, warp = tid >> 5;
    float* bufA = mbuf; float* bufB = mbuf + 4 * C; float* acc = mbuf + 8 * C;
    part = warp_sum(part);
    if (lane == 0) s_wpart[warp] = part;
    __syncthreads();
    const int dims[6] = {C, 2 * C, 4 * C, 2 * C, C, 1};
    const float* wp = mlp;
    float* in = bufA; float* out = bufB;
    for (int l = 0; l < (mlp ? 5 : 0); ++l) {
        const int cin = dims[l], cout = dims[l + 1];
        dense_layer(in, wp, wp + (size_t)cin * cout, cin, cout, l == 4, acc, out, tid);
        if constexpr (KEEP) for (int j = tid; j < cout; j += STEP_THREADS) keep[mlp_act_off(l + 1, C) + j] = out[j];
        wp += (size_t)cin * cout + cout;
        float* tmp = in; in = out; out = tmp;
        __syncthreads();
    }
    // bundlenet.py:249,253: base * ||rbar||^(2 + h); legacy/ba.py:280: ||rbar||^(1 + h); no MLP (legacy/ba.py:190): h = 0
    if (tid == 0) {
        float norm2 = 0.f;
        for (int wq = 0; wq < STEP_WARPS; ++wq) norm2 += s_wpart[wq];               // fixed order
        *s_lam = base * powf(sqrtf(norm2), exp0 + (mlp ? in[0] : 0.f)); *lambda_out = *s_lam;
        if constexpr (KEEP) keep[mlp_norm_off(C)] = sqrtf(norm2);
    }
    __syncthreads();
    return *s_lam;
}

// Blocked Cholesky of the lower triangle A[0:P][0:P] with the right-hand side as row P (afterwards A[P][:] = y = L^-1 g), then the back
// substitution L^T x = y into xs [P].  FULL: square storage with row pitch (P + 1) | 1; else packed.  dinv [P], dots [STEP_NB] scratch.
// A non-positive pivot sets bit 1 of *s_flag (the step is skipped by the caller).  All STEP_THREADS threads call it.
template <typename S, bool FULL>
__device__ __forceinline__ void step_cholesky_solve(S* A, int P, S* xs, S* dinv, S* dots, int* s_flag, int tid)
{
    const int lane = tid & 31, warp = tid >> 5;
    const int LD = (P + 1) | 1;
    auto IX = [&](int i, int k) -> int { return FULL ? i * LD + k : i * (i + 1) / 2 + k; };
    for (int j0 = 0; j0 < P; j0 += STEP_NB) {
        const int jb = min(STEP_NB, P - j0);
        // Panel: thread t owns row j0 + t (the block's own rows first, then the rows below, then the rhs row P).  EVERY owner factors the 8x8 diagonal
        // block redundantly in registers (36 independent loads, then a register-only chain) instead of waiting for one thread to do it through
        // shared memory (measured: that serial section and its barrier were 37 % of the kernel), then solves its own row against it.
        {
            const int i = j0 + tid;
            const bool owner = i <= P;
            S L[STEP_NB][STEP_NB], row[STEP_NB], Linv[STEP_NB];
            if (owner) {
#pragma unroll
                for (int r = 0; r < STEP_NB; ++r)
#pragma unroll
                    for (int c = 0; c < STEP_NB; ++c) L[r][c] = (c <= r && r < jb) ? A[IX(j0 + r, j0 + c)] : (S)(r == c ? 1 : 0);
#pragma unroll
                for (int c = 0; c < STEP_NB; ++c) row[c] = (c < jb && (tid >= jb || c <= tid)) ? A[IX(i, j0 + c)] : (S)0;
            }
            __syncthreads();                                         // every owner has read the block before its rows are overwritten
            if (owner) {
                bool notpd = false;
#pragma unroll
                for (int c = 0; c < STEP_NB; ++c) {                  // unblocked Cholesky of the block, registers only
                    S d = L[c][c];
#pragma unroll
                    for (int m = 0; m < STEP_NB; ++m) if (m < c) d -= L[c][m] * L[c][m];
                    if (c < jb && !(d > (S)0)) { notpd = true; d = (S)1; }
                    const S inv = rsqrt(d), ld = d * inv;                // one reciprocal square root per column; no divisions anywhere on the path
                    L[c][c] = ld; Linv[c] = inv;
#pragma unroll
                    for (int r = 0; r < STEP_NB; ++r) {
                        if (r > c) {
                            S v = L[r][c];
#pragma unroll
                            for (int m = 0; m < STEP_NB; ++m) if (m < c) v -= L[r][m] * L[c][m];
                            L[r][c] = v * inv;
                        }
                    }
                }
                if (tid == 0 && notpd) *s_flag |= 1;
                if (tid < jb) {                                      // a block row: its part of the factor
#pragma unroll
                    for (int c = 0; c < STEP_NB; ++c) if (c <= tid) { S v = (S)0;
#pragma unroll
                        for (int r = 0; r < STEP_NB; ++r) if (r == tid) v = L[r][c];
                        A[IX(i, j0 + c)] = v; }
#pragma unroll
                    for (int c = 0; c < STEP_NB; ++c) if (c == tid) dinv[j0 + c] = Linv[c];
                } else {                                             // a row below (or the rhs row): L21[i][:] = A21[i][:] L11^-T
#pragma unroll
                    for (int c = 0; c < STEP_NB; ++c) {
                        if (c < jb) {
                            S v = row[c];
#pragma unroll
                            for (int m = 0; m < STEP_NB; ++m) if (m < c) v -= row[m] * L[c][m];
                            row[c] = v * Linv[c];
                        }
                    }
#pragma unroll
                    for (int c = 0; c < STEP_NB; ++c) if (c < jb) A[IX(i, j0 + c)] = row[c];
                }
            }
        }
        __syncthreads();
        for (int i = j0 + jb + warp; i <= P; i += STEP_WARPS) {      // trailing update, warp per row, lanes over columns
            S li[STEP_NB];
#pragma unroll
            for (int c = 0; c < STEP_NB; ++c) li[c] = (c < jb) ? A[IX(i, j0 + c)] : (S)0;
            const int kend = (i == P) ? P - 1 : i;
            for (int k0 = j0 + jb; k0 <= kend; k0 += 128) {         // 4 independent column chunks in flight (no store between their loads)
                S sacc[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int k = k0 + 32 * q + lane;
                    S sv = (S)0;
                    if (k <= kend) {
#pragma unroll
                        for (int c = 0; c < STEP_NB; ++c) if (c < jb) sv += li[c] * A[IX(k, j0 + c)];
                    }
                    sacc[q] = sv;
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) { const int k = k0 + 32 * q + lane; if (k <= kend) A[IX(i, k)] -= sacc[q]; }
            }
        }
        __syncthreads();
    }

    // back substitution L^T x = y, panels from the bottom
    const int npan = (P + STEP_NB - 1) / STEP_NB;
    for (int pnl = npan - 1; pnl >= 0; --pnl) {
        const int j0 = pnl * STEP_NB, jb = min(STEP_NB, P - j0);
        if (warp < jb) {                                             // dots[c] = sum_{i >= j0+jb} L[i][j0+c] x[i]
            S s = (S)0;
            for (int i = j0 + jb + lane; i < P; i += 32) s += A[IX(i, j0 + warp)] * xs[i];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) dots[warp] = s;
        }
        __syncthreads();
        if (tid == 0) {                                              // 8x8 triangle in registers (independent loads first)
            S L[STEP_NB][STEP_NB], y[STEP_NB], x[STEP_NB];
#pragma unroll
            for (int r = 0; r < STEP_NB; ++r)
#pragma unroll
                for (int c = 0; c < STEP_NB; ++c) L[r][c] = (c <= r && r < jb) ? A[IX(j0 + r, j0 + c)] : (S)(r == c ? 1 : 0);
#pragma unroll
            for (int c = 0; c < STEP_NB; ++c) y[c] = (c < jb) ? A[IX(P, j0 + c)] - dots[c] : (S)0;
#pragma unroll
            for (int c = STEP_NB - 1; c >= 0; --c) {
                S v = y[c];
#pragma unroll
                for (int m = 0; m < STEP_NB; ++m) if (m > c) v -= L[m][c] * x[m];
                x[c] = v * (c < jb ? dinv[j0 + c] : (S)1);
            }
#pragma unroll
            for (int c = 0; c < STEP_NB; ++c) if (c < jb) xs[j0 + c] = x[c];
        }
        __syncthreads();
    }
}

// Adjoint of the damped solve delta = Ht^-1 g, Ht = H + diag(damp (diag H + eps)) lambda, given u = Ht^-1 ddelta (bundlenet.py:264-267):
//   dH = -u delta^T with the factor (1 + lambda) on the damped diagonal, dg = u, dlambda = -sum_{i < ndamped} u_i delta_i (H_ii + eps).
// u, dl (= delta) [P] in shared memory, Hb the pair's [P,P] H; flag != 0 (the forward skipped the step): every output 0.  All STEP_THREADS
// threads call it; dlambda is summed in double in a fixed order (bit-reproducible) and returned in thread 0.
template <typename S>
__device__ __forceinline__ float solve_adjoint_outputs(const S* u, const S* dl, const float* __restrict__ Hb, int P, int ndamped, float eps,
                                                       float lam, int flag, float* __restrict__ dHb, float* __restrict__ dgb, double* s_part,
                                                       int tid)
{
    double part = 0.0;
    for (int i = tid; i < P * P; i += STEP_THREADS) {
        const int rr = i / P, cc = i - rr * P;
        float v = 0.f;
        if (!flag) {
            double t = -(double)u[rr] * (double)dl[cc];
            if (rr == cc && rr < ndamped) { part += t * ((double)Hb[(size_t)rr * P + rr] + (double)eps); t *= 1.0 + (double)lam; }
            v = (float)t;
        }
        dHb[i] = v;
    }
    for (int i = tid; i < P; i += STEP_THREADS) dgb[i] = flag ? 0.f : (float)u[i];
    part += __shfl_xor_sync(0xffffffffu, part, 16); part += __shfl_xor_sync(0xffffffffu, part, 8); part += __shfl_xor_sync(0xffffffffu, part, 4);
    part += __shfl_xor_sync(0xffffffffu, part, 2); part += __shfl_xor_sync(0xffffffffu, part, 1);
    if ((tid & 31) == 0) s_part[tid >> 5] = part;
    __syncthreads();
    double dlam = 0.0;
    if (tid == 0)
        for (int wq = 0; wq < STEP_WARPS; ++wq) dlam += s_part[wq];
    return flag ? 0.f : (float)dlam;
}

// R' = exp(w) R, T' = V(w) t + exp(w) T in double (bundlenet.py:269-275) for one pair: dl = (w, t), Rb [3,3], Tb [3] -> Ro, To (may alias).
// skew: the skew matrix V is built from, when it is not the pair's own [w]x (the batch-interleaved one of bundlenet.py:45).
__device__ __forceinline__ void se3_update(const double* dl, const StepMode& mode, const float* Rb, const float* Tb, float* Ro, float* To,
                                           const double* skew = nullptr)
{
    const double wx = dl[0], wy = dl[1], wz = dl[2], tx = dl[3], ty = dl[4], tz = dl[5];
    const double th_raw = sqrt(wx * wx + wy * wy + wz * wz);
    const double th = mode.clamp_theta ? fmax(th_raw, 1e-6) : fmax(th_raw, 1e-300);      // AngleaAxisRotation (bundlenet.py:17-37; legacy/ba.py:60-80 has no clamp)
    const double kx = wx / th, ky = wy / th, kz = wz / th, c = cos(th), s = sin(th), oc = 1.0 - c;
    const double dr[9] = {c + kx * kx * oc,      kx * ky * oc - kz * s, ky * s + kx * kz * oc,
                          kz * s + kx * ky * oc, c + ky * ky * oc,      -kx * s + ky * kz * oc,
                          -ky * s + kx * kz * oc, kx * s + ky * kz * oc, c + kz * kz * oc};
    double ca, cb;                                               // VMatrix (bundlenet.py:39-46), series below 1e-4
    if (th_raw < 1e-4) { ca = 0.5 - th_raw * th_raw / 24.0; cb = 1.0 / 6.0 - th_raw * th_raw / 120.0; }
    else { ca = (1.0 - cos(th_raw)) / (th_raw * th_raw); cb = (th_raw - sin(th_raw)) / (th_raw * th_raw * th_raw); }
    const double own[9] = {0, -wz, wy, wz, 0, -wx, -wy, wx, 0};
    const double* sk = skew ? skew : own;
    double V[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
        const double sk2 = sk[i * 3] * sk[j] + sk[i * 3 + 1] * sk[3 + j] + sk[i * 3 + 2] * sk[6 + j];
        V[i * 3 + j] = ((i == j) ? 1.0 : 0.0) + ca * sk[i * 3 + j] + cb * sk2;
    }
    double Rin[9], Tin[3];
    for (int q = 0; q < 9; ++q) Rin[q] = Rb[q];
    for (int q = 0; q < 3; ++q) Tin[q] = Tb[q];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j)
            Ro[i * 3 + j] = (float)(dr[i * 3] * Rin[j] + dr[i * 3 + 1] * Rin[3 + j] + dr[i * 3 + 2] * Rin[6 + j]);
        const double vt = mode.use_vmatrix ? (V[i * 3] * tx + V[i * 3 + 1] * ty + V[i * 3 + 2] * tz) : dl[3 + i];     // legacy/ba.py:213: T' = t + dr T
        To[i] = (float)(vt + dr[i * 3] * Tin[0] + dr[i * 3 + 1] * Tin[1] + dr[i * 3 + 2] * Tin[2]);
    }
}

}  // namespace banet
