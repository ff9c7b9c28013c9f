// Backward of the per-pair SE(3) update (R' = exp(w) R, T' = V(w) t + exp(w) T; bundlenet.py:269-275) by forward-mode dual numbers in double,
// shared by lm_bwd.cu (thread per pair) and lm_window_batch.cu (thread per frame of a window).  Force-inlined: moving it here left
// pose_update_bwd_kernel's floating-point instructions and its outputs as they were.
#pragma once
#include "common.cuh"

namespace banet {

struct Dual3 {                                   // value + derivative along the three components of w
    double v, d[3];
    __device__ Dual3() : v(0) { d[0] = d[1] = d[2] = 0; }
    __device__ Dual3(double x) : v(x) { d[0] = d[1] = d[2] = 0; }
};
__device__ inline Dual3 operator+(const Dual3& a, const Dual3& b) { Dual3 r; r.v = a.v + b.v; for (int i = 0; i < 3; ++i) r.d[i] = a.d[i] + b.d[i]; return r; }
__device__ inline Dual3 operator-(const Dual3& a, const Dual3& b) { Dual3 r; r.v = a.v - b.v; for (int i = 0; i < 3; ++i) r.d[i] = a.d[i] - b.d[i]; return r; }
__device__ inline Dual3 operator-(const Dual3& a) { Dual3 r; r.v = -a.v; for (int i = 0; i < 3; ++i) r.d[i] = -a.d[i]; return r; }
__device__ inline Dual3 operator*(const Dual3& a, const Dual3& b) { Dual3 r; r.v = a.v * b.v; for (int i = 0; i < 3; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i]; return r; }
__device__ inline Dual3 operator/(const Dual3& a, const Dual3& b) { Dual3 r; r.v = a.v / b.v; for (int i = 0; i < 3; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) / b.v; return r; }
__device__ inline Dual3 dsin(const Dual3& a) { Dual3 r; r.v = sin(a.v); const double c = cos(a.v); for (int i = 0; i < 3; ++i) r.d[i] = c * a.d[i]; return r; }
__device__ inline Dual3 dcos(const Dual3& a) { Dual3 r; r.v = cos(a.v); const double s = -sin(a.v); for (int i = 0; i < 3; ++i) r.d[i] = s * a.d[i]; return r; }

// dl = (w, t) of one pair, Rb [3,3], Tb [3], gradients gRb, gTb of R', T' -> ddl [6] = dL/d(w, t), dRb [3,3], dTb [3]
__device__ __forceinline__ void pose_update_bwd_one(const double* dl, const float* Rb, const float* Tb, const float* gRb, const float* gTb,
                                                    float* ddl, float* dRb, float* dTb)
{
    Dual3 w[3];
    for (int i = 0; i < 3; ++i) { w[i].v = dl[i]; w[i].d[i] = 1.0; }
    const Dual3 th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    Dual3 thr; thr.v = sqrt(th2.v);
    if (thr.v > 1e-150) for (int i = 0; i < 3; ++i) thr.d[i] = th2.d[i] / (2.0 * thr.v);
    Dual3 th = thr; if (thr.v < 1e-6) th = Dual3(1e-6);                   // AngleaAxisRotation clamps theta (bundlenet.py:20)
    const Dual3 kx = w[0] / th, ky = w[1] / th, kz = w[2] / th, c = dcos(th), s = dsin(th), oc = Dual3(1.0) - c;
    const Dual3 dr[9] = {c + kx * kx * oc, kx * ky * oc - kz * s, ky * s + kx * kz * oc,
                         kz * s + kx * ky * oc, c + ky * ky * oc, ky * kz * oc - kx * s,
                         kx * kz * oc - ky * s, kx * s + ky * kz * oc, c + kz * kz * oc};
    Dual3 ca, cb;
    if (thr.v < 1e-4) { ca = Dual3(0.5) - th2 / Dual3(24.0); cb = Dual3(1.0 / 6.0) - th2 / Dual3(120.0); }
    else { ca = (Dual3(1.0) - dcos(thr)) / th2; cb = (thr - dsin(thr)) / (th2 * thr); }
    const Dual3 zero(0.0);
    const Dual3 sk[9] = {zero, -w[2], w[1], w[2], zero, -w[0], -w[1], w[0], zero};
    Dual3 V[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
        const Dual3 sk2 = sk[i * 3] * sk[j] + sk[i * 3 + 1] * sk[3 + j] + sk[i * 3 + 2] * sk[6 + j];
        V[i * 3 + j] = Dual3(i == j ? 1.0 : 0.0) + ca * sk[i * 3 + j] + cb * sk2;
    }
    double Rin[9], Tin[3], gR[9], gT[3];
    for (int q = 0; q < 9; ++q) { Rin[q] = Rb[q]; gR[q] = gRb[q]; }
    for (int q = 0; q < 3; ++q) { Tin[q] = Tb[q]; gT[q] = gTb[q]; }
    for (int k = 0; k < 3; ++k) {
        double acc = 0.0;
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) {
                double dRij = 0.0;
                for (int m = 0; m < 3; ++m) dRij += dr[i * 3 + m].d[k] * Rin[m * 3 + j];
                acc += gR[i * 3 + j] * dRij;
            }
            double dTi = 0.0;
            for (int m = 0; m < 3; ++m) dTi += V[i * 3 + m].d[k] * dl[3 + m] + dr[i * 3 + m].d[k] * Tin[m];
            acc += gT[i] * dTi;
        }
        ddl[k] = (float)acc;
    }
    for (int m = 0; m < 3; ++m) {
        double a = 0.0;
        for (int i = 0; i < 3; ++i) a += V[i * 3 + m].v * gT[i];
        ddl[3 + m] = (float)a;
    }
    for (int i = 0; i < 3; ++i) {                                          // dR = dr^T gR', dT = dr^T gT'
        for (int j = 0; j < 3; ++j) {
            double a = 0.0;
            for (int m = 0; m < 3; ++m) a += dr[m * 3 + i].v * gR[m * 3 + j];
            dRb[i * 3 + j] = (float)a;
        }
        double a = 0.0;
        for (int m = 0; m < 3; ++m) a += dr[m * 3 + i].v * gT[m];
        dTb[i] = (float)a;
    }
}

}  // namespace banet
