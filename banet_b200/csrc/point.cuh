// Per-point code of the fp32 SIMT build kernels: lm_build_kernel (lm_build.cu), lm_build_bwd_kernel (lm_bwd.cu), the keyframe build and
// its backward (lm_window_key.cu), and the feature-metric cost and its backward (lm_cost.cu).  Each piece is one step of one point,
// computed exactly as every one of those kernels needs it; the tile and frame loops, the slot layouts and the way each kernel stores or
// commits its sums stay in the kernels.
#pragma once
#include "common.cuh"
#include "features.cuh"

namespace banet {

__device__ __forceinline__ int reflect1(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }     // tf.pad REFLECT by one (bundlenet.py:97)
__device__ __forceinline__ float sgn(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }

template <int G> __device__ __forceinline__ void lds_group(const float* p, float* out);
template <> __device__ __forceinline__ void lds_group<1>(const float* p, float* o) { o[0] = p[0]; }
template <> __device__ __forceinline__ void lds_group<2>(const float* p, float* o) {
    float2 v = *reinterpret_cast<const float2*>(p); o[0] = v.x; o[1] = v.y; }
template <> __device__ __forceinline__ void lds_group<4>(const float* p, float* o) {
    float4 v = *reinterpret_cast<const float4*>(p); o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w; }

// one group of VEC channels; TF: element type of the feature loads (float, or bf16 widened exactly on load); the |diff| sums in smem are always fp32
template <int VEC, typename TF = float> struct ChanVec;
template <> struct ChanVec<4> {
    float v[4];
    __device__ __forceinline__ void load(const float* p) { float4 t = __ldg(reinterpret_cast<const float4*>(p)); v[0]=t.x; v[1]=t.y; v[2]=t.z; v[3]=t.w; }
    __device__ __forceinline__ void load_stream(const float* p) { float4 t = ld_stream_f4(p); v[0]=t.x; v[1]=t.y; v[2]=t.z; v[3]=t.w; }
    __device__ __forceinline__ void load_smem(const float* p) { float4 t = *reinterpret_cast<const float4*>(p); v[0]=t.x; v[1]=t.y; v[2]=t.z; v[3]=t.w; }
    __device__ __forceinline__ void store_smem(float* p) const { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};
template <> struct ChanVec<1> {
    float v[1];
    __device__ __forceinline__ void load(const float* p) { v[0] = __ldg(p); }
    __device__ __forceinline__ void load_stream(const float* p) { v[0] = ld_stream_f1(p); }
    __device__ __forceinline__ void load_smem(const float* p) { v[0] = p[0]; }
    __device__ __forceinline__ void store_smem(float* p) const { p[0] = v[0]; }
};
template <> struct ChanVec<4, bf16> {
    float v[4];
    __device__ __forceinline__ void set(uint2 t) { v[0] = bf16_lo(t.x); v[1] = bf16_hi(t.x); v[2] = bf16_lo(t.y); v[3] = bf16_hi(t.y); }
    __device__ __forceinline__ void load(const bf16* p) { set(__ldg(reinterpret_cast<const uint2*>(p))); }
    __device__ __forceinline__ void load_stream(const bf16* p) { set(ld_stream_bf4(p)); }
};
template <> struct ChanVec<1, bf16> {
    float v[1];
    __device__ __forceinline__ void load(const bf16* p) { v[0] = ldg_feat(p); }
    __device__ __forceinline__ void load_stream(const bf16* p) { v[0] = ld_stream_bf1(p); }
};

// ---- forward --------------------------------------------------------------------------------------------------------------------------
// b.W of one staged basis row (KP entries, a multiple of 4, padded with zeros) in four partial sums
template <int KP>
__device__ __forceinline__ float basis_dot(const float* brow, const float* sW) {
    float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
#pragma unroll 4
    for (int k = 0; k < KP; k += 4) {
        const float4 bv = *reinterpret_cast<const float4*>(brow + k);
        const float4 wv = *reinterpret_cast<const float4*>(sW + k);
        d0 = fmaf(bv.x, wv.x, d0); d1 = fmaf(bv.y, wv.y, d1);
        d2 = fmaf(bv.z, wv.z, d2); d3 = fmaf(bv.w, wv.w, d3);
    }
    return (d0 + d1) + (d2 + d3);
}

// The warp of one point (bundlenet.py:208-224): ray p at depth Dt through pose = R (9) | T (3) | fx fy ox oy.  r = R p, (x, y) = X / Z,
// Y / Z with X = r Dt + T, iZ = 1 / Z, and the pixel (u, v).
struct Projection {
    float rx, ry, rz, x, y, iZ, u, v;
    __device__ __forceinline__ Projection(const float* pose, float p0, float p1, float p2, float Dt) {
        rx = pose[0] * p0 + pose[1] * p1 + pose[2] * p2;
        ry = pose[3] * p0 + pose[4] * p1 + pose[5] * p2;
        rz = pose[6] * p0 + pose[7] * p1 + pose[8] * p2;
        const float X = rx * Dt + pose[9], Y = ry * Dt + pose[10], Z = rz * Dt + pose[11];
        x = X / Z; y = Y / Z; iZ = 1.0f / Z;
        u = pose[12] * x + pose[14]; v = pose[13] * y + pose[15];
    }
    // reference mask (bundlenet.py:231): not(px<0 | px>w-1 | py<0 | py>h-1); non-finite projections are masked too
    __device__ __forceinline__ bool in_bounds(int h, int w) const {
        return (u >= 0.f) && (u <= (float)(w - 1)) && (v >= 0.f) && (v <= (float)(h - 1)) && isfinite(iZ);
    }
};

// The bilinear taps of an in-bounds pixel: corner (x0, y0), the far corner clamped to the image, the fractions dx, dy and the four weights
// (tap bit 0: x0 / x1, bit 1: y0 / y1)
struct Taps {
    int x0, y0, x1, y1;
    float dx, dy, w00, w01, w10, w11;
    __device__ __forceinline__ Taps(int x0_, int y0_, float dx_, float dy_, int h, int w)
        : x0(x0_), y0(y0_), x1(min(x0_ + 1, w - 1)), y1(min(y0_ + 1, h - 1)), dx(dx_), dy(dy_),
          w00((1.f - dx_) * (1.f - dy_)), w01(dx_ * (1.f - dy_)), w10((1.f - dx_) * dy_), w11(dx_ * dy_) {}
};
__device__ __forceinline__ void tap_corner(float u, float v, int& x0, int& y0, float& dx, float& dy) {
    const float fu = floorf(u), fv = floorf(v);
    x0 = (int)fu; y0 = (int)fv; dx = u - fu; dy = v - fv;
}
__device__ __forceinline__ Taps taps_at(float u, float v, int h, int w) {
    int x0, y0; float dx, dy;
    tap_corner(u, v, x0, y0, dx, dy);
    return Taps(x0, y0, dx, dy, h, w);
}

// M = G^T G (m11, m12, m22) and q = G^T d (q1, q2) of one point, and s = d^T d (the argument of its robust loss)
struct PointMQ { float m11, m12, m22, q1, q2, s; };

// The feature gather of one point (bundlenet.py:230-239) from the frame's conv2 map img with c2 channels per texel: [F2 | gx | gy] (c2 = 3C),
// or F2 only (fly, c2 = C: the gradients are central differences with REFLECT-by-one borders at each tap, bundlenet.py:92-100).
template <typename TF>
struct TapGather {
    const TF *img, *t00, *t01, *t10, *t11;
    int x0, x1, y0, y1, h, w, C, c2;
    float w00, w01, w10, w11;
    __device__ __forceinline__ TapGather(const TF* img_, const Taps& tp, int h_, int w_, int C_, int c2_)
        : img(img_), t00(img_ + ((size_t)tp.y0 * w_ + tp.x0) * c2_), t01(img_ + ((size_t)tp.y0 * w_ + tp.x1) * c2_),
          t10(img_ + ((size_t)tp.y1 * w_ + tp.x0) * c2_), t11(img_ + ((size_t)tp.y1 * w_ + tp.x1) * c2_),
          x0(tp.x0), x1(tp.x1), y0(tp.y0), y1(tp.y1), h(h_), w(w_), C(C_), c2(c2_), w00(tp.w00), w01(tp.w01), w10(tp.w10), w11(tp.w11) {}
    // channels [c, c + VEC), f1 holding conv1's: accumulates M, q, s into mq and |d| into the fp32 sums rb[c, c + VEC) in shared memory
    template <int VEC>
    __device__ __forceinline__ void group(const ChanVec<VEC, TF>& f1, bool fly, int c, float* rb, PointMQ& mq) const {
        ChanVec<VEC, TF> a00, a01, a10, a11;
        ChanVec<VEC> gx, gy;
        a00.load(t00 + c); a01.load(t01 + c); a10.load(t10 + c); a11.load(t11 + c);
        if (!fly) {
            ChanVec<VEC, TF> g00, g01, g10, g11;
            g00.load(t00 + C + c); g01.load(t01 + C + c); g10.load(t10 + C + c); g11.load(t11 + C + c);
#pragma unroll
            for (int u = 0; u < VEC; ++u) gx.v[u] = w00 * g00.v[u] + w01 * g01.v[u] + w10 * g10.v[u] + w11 * g11.v[u];
            g00.load(t00 + 2 * C + c); g01.load(t01 + 2 * C + c); g10.load(t10 + 2 * C + c); g11.load(t11 + 2 * C + c);
#pragma unroll
            for (int u = 0; u < VEC; ++u) gy.v[u] = w00 * g00.v[u] + w01 * g01.v[u] + w10 * g10.v[u] + w11 * g11.v[u];
        } else {
#pragma unroll
            for (int u = 0; u < VEC; ++u) { gx.v[u] = 0.f; gy.v[u] = 0.f; }
            const int xs[2] = {x0, x1}, ys[2] = {y0, y1};
            const float wt[4] = {w00, w01, w10, w11};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int xx = xs[k & 1], yy = ys[k >> 1];
                ChanVec<VEC, TF> e, wv, s, nn;
                e.load(img + ((size_t)yy * w + reflect1(xx + 1, w)) * c2 + c);
                wv.load(img + ((size_t)yy * w + reflect1(xx - 1, w)) * c2 + c);
                s.load(img + ((size_t)reflect1(yy + 1, h) * w + xx) * c2 + c);
                nn.load(img + ((size_t)reflect1(yy - 1, h) * w + xx) * c2 + c);
#pragma unroll
                for (int u = 0; u < VEC; ++u) {
                    gx.v[u] = fmaf(wt[k], 0.5f * (e.v[u] - wv.v[u]), gx.v[u]);
                    gy.v[u] = fmaf(wt[k], 0.5f * (s.v[u] - nn.v[u]), gy.v[u]);
                }
            }
        }
        ChanVec<VEC> ra;
        ra.load_smem(rb + c);
#pragma unroll
        for (int u = 0; u < VEC; ++u) {
            const float f2 = w00 * a00.v[u] + w01 * a01.v[u] + w10 * a10.v[u] + w11 * a11.v[u];
            const float d = f1.v[u] - f2;
            mq.m11 = fmaf(gx.v[u], gx.v[u], mq.m11); mq.m12 = fmaf(gx.v[u], gy.v[u], mq.m12); mq.m22 = fmaf(gy.v[u], gy.v[u], mq.m22);
            mq.q1 = fmaf(gx.v[u], d, mq.q1); mq.q2 = fmaf(gy.v[u], d, mq.q2); mq.s = fmaf(d, d, mq.s);
            ra.v[u] += fabsf(d);
        }
        ra.store_smem(rb + c);
    }
};

// b.W of a staged basis row padded to KP (a runtime value of padded_K) in basis_dot<KP>'s own arithmetic: kernels that take every K in
// one instantiation get the build's depth, and therefore its mask, bit for bit
__device__ __forceinline__ float basis_dot_padded(const float* brow, const float* sW, int KP) {
    switch (KP) {
        case 16:  return basis_dot<16>(brow, sW);
        case 32:  return basis_dot<32>(brow, sW);
        case 64:  return basis_dot<64>(brow, sW);
        case 128: return basis_dot<128>(brow, sW);
        default:  return basis_dot<256>(brow, sW);
    }
}

// The value-only sample of one point (the feature-metric cost, lm_cost.cu): F2 at the four taps, the first C channels of each texel of a
// map with c2 channels per texel (3C: the gradient channels are never read; C: F2 only, no stencil).  d_c = conv1_c - F2(u, v)_c with the
// bilinear weights in TapGather's order.  Offsets are elements from the pair's map, so the same taps address conv2 and dconv2.
struct ValueTaps {
    size_t o00, o01, o10, o11;
    float w00, w01, w10, w11, dx, dy;
    __device__ __forceinline__ ValueTaps(const Taps& tp, int w, int c2)
        : o00(((size_t)tp.y0 * w + tp.x0) * c2), o01(((size_t)tp.y0 * w + tp.x1) * c2), o10(((size_t)tp.y1 * w + tp.x0) * c2),
          o11(((size_t)tp.y1 * w + tp.x1) * c2), w00(tp.w00), w01(tp.w01), w10(tp.w10), w11(tp.w11), dx(tp.dx), dy(tp.dy) {}
    // channels [c, c + VEC), f1 holding conv1's: accumulates d_c^2 into s
    template <int VEC, typename TF>
    __device__ __forceinline__ void squares(const TF* img, const ChanVec<VEC, TF>& f1, int c, float& s) const {
        ChanVec<VEC, TF> a00, a01, a10, a11;
        a00.load(img + o00 + c); a01.load(img + o01 + c); a10.load(img + o10 + c); a11.load(img + o11 + c);
#pragma unroll
        for (int u = 0; u < VEC; ++u) {
            const float d = f1.v[u] - (w00 * a00.v[u] + w01 * a01.v[u] + w10 * a10.v[u] + w11 * a11.v[u]);
            s = fmaf(d, d, s);
        }
    }
    // channel c alone (lanes over channels): d_c, and the tap values in t
    template <typename TF>
    __device__ __forceinline__ float residual(const TF* img, const TF* c1, int c, float t[4]) const {
        t[0] = ldg_feat(img + o00 + c); t[1] = ldg_feat(img + o01 + c); t[2] = ldg_feat(img + o10 + c); t[3] = ldg_feat(img + o11 + c);
        return ldg_feat(c1 + c) - (w00 * t[0] + w01 * t[1] + w10 * t[2] + w11 * t[3]);
    }
    // the adjoint of channel c's sample, given df = dL/dF2_c and the tap values t: w_tau df into the taps of dimg (atomics), and the
    // gradient of the pixel coordinates from the tap differences added to (du, dv)
    __device__ __forceinline__ void adjoint(float* dimg, int c, const float t[4], float df, float& du, float& dv) const {
        atomicAdd(dimg + o00 + c, w00 * df); atomicAdd(dimg + o01 + c, w01 * df); atomicAdd(dimg + o10 + c, w10 * df); atomicAdd(dimg + o11 + c, w11 * df);
        du += df * ((1.f - dy) * (t[1] - t[0]) + dy * (t[3] - t[2]));
        dv += df * ((1.f - dx) * (t[2] - t[0]) + dx * (t[3] - t[1]));
    }
};

// CameraJacobianMatrix, negated (bundlenet.py:58-60): the rows a0, a1 of Jc
__device__ __forceinline__ void camera_jacobian(float fx, float fy, float x, float y, float iZ, float a0[6], float a1[6]) {
    a0[0] = -fx * (x * y); a0[1] = -fx * (-1.f - x * x); a0[2] = -fx * y; a0[3] = -fx * (-iZ); a0[4] = 0.f; a0[5] = -fx * (x * iZ);
    a1[0] = -fy * (1.f + y * y); a1[1] = -fy * (-(x * y)); a1[2] = -fy * (-x); a1[3] = 0.f; a1[4] = -fy * (-iZ); a1[5] = -fy * (y * iZ);
}
// DepthJacobianMatrix (bundlenet.py:69-70): jd = (jd0, jd1)
__device__ __forceinline__ void depth_jacobian(float fx, float fy, float rx, float ry, float rz, float x, float y, float iZ, float& jd0, float& jd1) {
    jd0 = fx * ((rx - rz * x) * iZ); jd1 = fy * ((ry - rz * y) * iZ);
}

// one point's camera block: the 21 entries of Jc^T M Jc (upper triangle, row-major) and the 6 of Jc^T q
__device__ __forceinline__ void pose_terms(const float a0[6], const float a1[6], const PointMQ& mq, float t[27]) {
    float ux[6], uy[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) { ux[i] = mq.m11 * a0[i] + mq.m12 * a1[i]; uy[i] = mq.m12 * a0[i] + mq.m22 * a1[i]; }
    int q = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int jj = i; jj < 6; ++jj) { t[q] = a0[i] * ux[jj] + a1[i] * uy[jj]; ++q; }
#pragma unroll
    for (int i = 0; i < 6; ++i) t[21 + i] = a0[i] * mq.q1 + a1[i] * mq.q2;
}
// one point's depth terms ext = v (6: Jc^T M jd), t (jd^T q), s (jd^T M jd): H_cd += v b^T, g_d += t b, H_dd += s b b^T
__device__ __forceinline__ void depth_terms(const float a0[6], const float a1[6], float jd0, float jd1, const PointMQ& mq, float ext[8]) {
    const float u0 = mq.m11 * jd0 + mq.m12 * jd1, u1 = mq.m12 * jd0 + mq.m22 * jd1;
#pragma unroll
    for (int i = 0; i < 6; ++i) ext[i] = a0[i] * u0 + a1[i] * u1;
    ext[6] = jd0 * mq.q1 + jd1 * mq.q2;
    ext[7] = jd0 * u0 + jd1 * u1;
}

// ---- backward ---------------------------------------------------------------------------------------------------------------------------
// Pixel coordinates of the four taps (bit 0: x0 / x1, bit 1: y0 / y1) and of their stencil neighbours in an F2-only map.
struct FlyTaps {
    int cx[2], ex[2], wx[2], cy[2], sy[2], ny[2];
    __device__ __forceinline__ FlyTaps(int x0, int x1, int y0, int y1, int h, int w) {
        cx[0] = x0; cx[1] = x1; cy[0] = y0; cy[1] = y1;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            ex[i] = reflect1(cx[i] + 1, w); wx[i] = reflect1(cx[i] - 1, w);
            sy[i] = reflect1(cy[i] + 1, h); ny[i] = reflect1(cy[i] - 1, h);
        }
    }
    // channel c of the tap values t, the tap x-gradients g and y-gradients k
    template <typename TF>
    __device__ __forceinline__ void load(const TF* img, int w, int C, int c, float t[4], float g[4], float k[4]) const {
#pragma unroll
        for (int tp = 0; tp < 4; ++tp) {
            const int xx = cx[tp & 1];
            const size_t row = (size_t)cy[tp >> 1] * w;
            t[tp] = ldg_feat(img + (row + xx) * C + c);
            g[tp] = 0.5f * (ldg_feat(img + (row + ex[tp & 1]) * C + c) - ldg_feat(img + (row + wx[tp & 1]) * C + c));
            k[tp] = 0.5f * (ldg_feat(img + ((size_t)sy[tp >> 1] * w + xx) * C + c) - ldg_feat(img + ((size_t)ny[tp >> 1] * w + xx) * C + c));
        }
    }
    // the adjoint of load for one channel: df on the values, dgx / dgy on the gradients, each tap weighted by wt
    __device__ __forceinline__ void scatter(float* dimg, int w, int C, int c, const float wt[4], float df, float dgx, float dgy) const {
#pragma unroll
        for (int tp = 0; tp < 4; ++tp) {
            const int xx = cx[tp & 1];
            const size_t row = (size_t)cy[tp >> 1] * w;
            const float hx = 0.5f * wt[tp] * dgx, hy = 0.5f * wt[tp] * dgy;
            atomicAdd(dimg + (row + xx) * C + c, wt[tp] * df);
            atomicAdd(dimg + (row + ex[tp & 1]) * C + c, hx); atomicAdd(dimg + (row + wx[tp & 1]) * C + c, -hx);
            atomicAdd(dimg + ((size_t)sy[tp >> 1] * w + xx) * C + c, hy); atomicAdd(dimg + ((size_t)ny[tp >> 1] * w + xx) * C + c, -hy);
        }
    }
};

// Pass 1 of the backward, lanes over channels: M, q of one point, summed over the warp, and s as this lane's partial (a caller that uses
// it sums it with warp_sum; one that does not leaves no trace of it in its code).  FLY: conv2 is F2 only (the gradients from the stencil
// at each tap); otherwise [F2 | gx | gy].
template <bool FLY, typename TF>
__device__ __forceinline__ PointMQ point_mq(const TF* img, const TF* c1, const Taps& tp, int h, int w, int C, int lane) {
    const int C3 = FLY ? C : 3 * C;
    const float w00 = tp.w00, w01 = tp.w01, w10 = tp.w10, w11 = tp.w11;
    const size_t o00 = ((size_t)tp.y0 * w + tp.x0) * C3, o01 = ((size_t)tp.y0 * w + tp.x1) * C3, o10 = ((size_t)tp.y1 * w + tp.x0) * C3, o11 = ((size_t)tp.y1 * w + tp.x1) * C3;
    float m11 = 0.f, m12 = 0.f, m22 = 0.f, q1 = 0.f, q2 = 0.f, s = 0.f;
    for (int c = lane; c < C; c += 32) {
        float f2, gx, gy;
        if constexpr (FLY) {
            const FlyTaps fly(tp.x0, tp.x1, tp.y0, tp.y1, h, w);
            float t[4], g[4], k[4];
            fly.load(img, w, C, c, t, g, k);
            f2 = w00 * t[0] + w01 * t[1] + w10 * t[2] + w11 * t[3];
            gx = w00 * g[0] + w01 * g[1] + w10 * g[2] + w11 * g[3];
            gy = w00 * k[0] + w01 * k[1] + w10 * k[2] + w11 * k[3];
        } else {
            f2 = w00 * ldg_feat(img + o00 + c) + w01 * ldg_feat(img + o01 + c) + w10 * ldg_feat(img + o10 + c) + w11 * ldg_feat(img + o11 + c);
            gx = w00 * ldg_feat(img + o00 + C + c) + w01 * ldg_feat(img + o01 + C + c) + w10 * ldg_feat(img + o10 + C + c) + w11 * ldg_feat(img + o11 + C + c);
            gy = w00 * ldg_feat(img + o00 + 2 * C + c) + w01 * ldg_feat(img + o01 + 2 * C + c) + w10 * ldg_feat(img + o10 + 2 * C + c) + w11 * ldg_feat(img + o11 + 2 * C + c);
        }
        const float d = ldg_feat(c1 + c) - f2;
        m11 = fmaf(gx, gx, m11); m12 = fmaf(gx, gy, m12); m22 = fmaf(gy, gy, m22); q1 = fmaf(gx, d, q1); q2 = fmaf(gy, d, q2); s = fmaf(d, d, s);
    }
    return PointMQ{warp_sum(m11), warp_sum(m12), warp_sum(m22), warp_sum(q1), warp_sum(q2), s};
}

// The adjoint of one point's 2 x (6+1) algebra.  With S = the symmetrised dL/dH and ghat = dL/dg, alpha = S_cd b, beta = S_dc^T b,
// eta = ghat_d . b, gamma = b^T S_dd b:
//   Y_c = Jc S_cc + jd beta^T      Y_d b = Jc alpha + jd gamma      z = Jc ghat_c + jd eta      Q = Y J^T (2x2)
struct PointAdjoint {
    float Yc0[6], Yc1[6], yb0, yb1, z0, z1, Q00, Q01, Q10, Q11;
    __device__ __forceinline__ PointAdjoint(const float a0[6], const float a1[6], float jd0, float jd1, const float* Scc, const float* sg,
                                            const float alpha[6], const float beta[6], float eta, float gamma) {
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            float s0 = jd0 * beta[i], s1 = jd1 * beta[i];
#pragma unroll
            for (int m = 0; m < 6; ++m) { s0 = fmaf(a0[m], Scc[m * 6 + i], s0); s1 = fmaf(a1[m], Scc[m * 6 + i], s1); }
            Yc0[i] = s0; Yc1[i] = s1;
        }
        float fb0 = 0.f, fb1 = 0.f;
        z0 = jd0 * eta; z1 = jd1 * eta;
#pragma unroll
        for (int m = 0; m < 6; ++m) { fb0 = fmaf(a0[m], alpha[m], fb0); fb1 = fmaf(a1[m], alpha[m], fb1); z0 = fmaf(a0[m], sg[m], z0); z1 = fmaf(a1[m], sg[m], z1); }
        yb0 = fb0 + jd0 * gamma; yb1 = fb1 + jd1 * gamma;
        Q00 = yb0 * jd0; Q01 = yb0 * jd1; Q10 = yb1 * jd0; Q11 = yb1 * jd1;
#pragma unroll
        for (int i = 0; i < 6; ++i) { Q00 = fmaf(Yc0[i], a0[i], Q00); Q01 = fmaf(Yc0[i], a1[i], Q01); Q10 = fmaf(Yc1[i], a0[i], Q10); Q11 = fmaf(Yc1[i], a1[i], Q11); }
    }
    // point weight w: dw = <Ghat, H_n> + <ghat, g_n> = 1/2 <M, Q> + q.z (H_n = J^T M J is symmetric, so this is exact for both S
    // conventions), returned.  Every adjoint that comes from Ghat, ghat is the point's times w: scaling M, q carries it to dJ and db, scaling
    // Q, z to dG and dd; the rhat sign(d) path is not weighted.  Unweighted: w = 1 and x * 1.0f is exact.
    __device__ __forceinline__ float weigh(float wn, PointMQ& mq) {
        const float dw = 0.5f * (mq.m11 * Q00 + mq.m12 * (Q01 + Q10) + mq.m22 * Q11) + (mq.q1 * z0 + mq.q2 * z1);
        mq.m11 *= wn; mq.m12 *= wn; mq.m22 *= wn; mq.q1 *= wn; mq.q2 *= wn;
        Q00 *= wn; Q01 *= wn; Q10 *= wn; Q11 *= wn; z0 *= wn; z1 *= wn;
        return dw;
    }
};

// dJ = M Y + q ghat^T: camera columns dJ0, dJ1, depth column dj0, dj1
__device__ __forceinline__ void jacobian_adjoint(const PointMQ& mq, const PointAdjoint& ad, const float* sg, float eta, float dJ0[6], float dJ1[6],
                                                 float& dj0, float& dj1) {
#pragma unroll
    for (int i = 0; i < 6; ++i) { dJ0[i] = mq.m11 * ad.Yc0[i] + mq.m12 * ad.Yc1[i] + mq.q1 * sg[i]; dJ1[i] = mq.m12 * ad.Yc0[i] + mq.m22 * ad.Yc1[i] + mq.q2 * sg[i]; }
    dj0 = mq.m11 * ad.yb0 + mq.m12 * ad.yb1 + mq.q1 * eta; dj1 = mq.m12 * ad.yb0 + mq.m22 * ad.yb1 + mq.q2 * eta;
}

// Pass 2 of the backward, lanes over channels: per channel c, dd_c = G_c z + rhat_c sign(d_c) (+ ds2 d_c, the robust weight's term
// 2 ds d_c; skipped when ds2 == 0) goes to put_dd(c, dd_c); the feature map's adjoint (taps of -dd_c on the values, dG_c = G_c Q + d_c z^T
// on the gradients) is scattered into dimg with atomics; returns the gradient (du, dv) of the pixel coordinates, summed over the warp.
template <bool FLY, typename TF, typename PutDd>
__device__ __forceinline__ void channel_adjoint(const TF* img, float* dimg, const TF* c1, const float* sRh, const Taps& tp, int h, int w, int C,
                                                int lane, const PointAdjoint& ad, float ds2, PutDd put_dd, float& du_out, float& dv_out) {
    const int C3 = FLY ? C : 3 * C;
    const float w00 = tp.w00, w01 = tp.w01, w10 = tp.w10, w11 = tp.w11, dx = tp.dx, dy = tp.dy;
    const float z0 = ad.z0, z1 = ad.z1, Q00 = ad.Q00, Q01 = ad.Q01, Q10 = ad.Q10, Q11 = ad.Q11;
    const size_t o00 = ((size_t)tp.y0 * w + tp.x0) * C3, o01 = ((size_t)tp.y0 * w + tp.x1) * C3, o10 = ((size_t)tp.y1 * w + tp.x0) * C3, o11 = ((size_t)tp.y1 * w + tp.x1) * C3;
    float du = 0.f, dv = 0.f;
    for (int c = lane; c < C; c += 32) {
        float t00, t01, t10, t11, g00, g01, g10, g11, k00, k01, k10, k11;
        if constexpr (FLY) {
            const FlyTaps fly(tp.x0, tp.x1, tp.y0, tp.y1, h, w);
            float t[4], g[4], k[4];
            fly.load(img, w, C, c, t, g, k);
            t00 = t[0]; t01 = t[1]; t10 = t[2]; t11 = t[3]; g00 = g[0]; g01 = g[1]; g10 = g[2]; g11 = g[3]; k00 = k[0]; k01 = k[1]; k10 = k[2]; k11 = k[3];
        } else {
            t00 = ldg_feat(img + o00 + c); t01 = ldg_feat(img + o01 + c); t10 = ldg_feat(img + o10 + c); t11 = ldg_feat(img + o11 + c);
            g00 = ldg_feat(img + o00 + C + c); g01 = ldg_feat(img + o01 + C + c); g10 = ldg_feat(img + o10 + C + c); g11 = ldg_feat(img + o11 + C + c);
            k00 = ldg_feat(img + o00 + 2 * C + c); k01 = ldg_feat(img + o01 + 2 * C + c); k10 = ldg_feat(img + o10 + 2 * C + c); k11 = ldg_feat(img + o11 + 2 * C + c);
        }
        const float f2 = w00 * t00 + w01 * t01 + w10 * t10 + w11 * t11;
        const float gx = w00 * g00 + w01 * g01 + w10 * g10 + w11 * g11;
        const float gy = w00 * k00 + w01 * k01 + w10 * k10 + w11 * k11;
        const float d = ldg_feat(c1 + c) - f2;
        float dd = gx * z0 + gy * z1 + sRh[c] * sgn(d);
        if (ds2 != 0.f) dd = fmaf(ds2, d, dd);
        const float dgx = gx * Q00 + gy * Q10 + d * z0, dgy = gx * Q01 + gy * Q11 + d * z1;
        put_dd(c, dd);
        const float df = -dd;
        if constexpr (FLY) {
            const float wt[4] = {w00, w01, w10, w11};
            const FlyTaps fly(tp.x0, tp.x1, tp.y0, tp.y1, h, w);
            fly.scatter(dimg, w, C, c, wt, df, dgx, dgy);
        } else {
            atomicAdd(dimg + o00 + c, w00 * df); atomicAdd(dimg + o01 + c, w01 * df); atomicAdd(dimg + o10 + c, w10 * df); atomicAdd(dimg + o11 + c, w11 * df);
            atomicAdd(dimg + o00 + C + c, w00 * dgx); atomicAdd(dimg + o01 + C + c, w01 * dgx); atomicAdd(dimg + o10 + C + c, w10 * dgx); atomicAdd(dimg + o11 + C + c, w11 * dgx);
            atomicAdd(dimg + o00 + 2 * C + c, w00 * dgy); atomicAdd(dimg + o01 + 2 * C + c, w01 * dgy); atomicAdd(dimg + o10 + 2 * C + c, w10 * dgy); atomicAdd(dimg + o11 + 2 * C + c, w11 * dgy);
        }
        du += df * ((1.f - dy) * (t01 - t00) + dy * (t11 - t10)) + dgx * ((1.f - dy) * (g01 - g00) + dy * (g11 - g10)) + dgy * ((1.f - dy) * (k01 - k00) + dy * (k11 - k10));
        dv += df * ((1.f - dx) * (t10 - t00) + dx * (t11 - t01)) + dgx * ((1.f - dx) * (g10 - g00) + dx * (g11 - g01)) + dgy * ((1.f - dx) * (k10 - k00) + dx * (k11 - k01));
    }
    du_out = warp_sum(du); dv_out = warp_sum(dv);
}

// The geometry backward of one point: from the pixel gradient (du, dv) and dJ, dj through the Jacobians and the projection to the camera-frame
// point (gX, gY, gZ), the depth (gDt) and the rotated ray (grx, gry, grz)
struct GeomGrad {
    float gX, gY, gZ, gDt, grx, gry, grz;
    __device__ __forceinline__ GeomGrad(const Projection& pr, float fx, float fy, float Dt, float du, float dv, const float dJ0[6], const float dJ1[6],
                                        float dj0, float dj1) {
        const float x = pr.x, y = pr.y, iZ = pr.iZ, rx = pr.rx, ry = pr.ry, rz = pr.rz;
        float gxx = fx * du, gyy = fy * dv, giZ = 0.f;                      // u = fx x + ox, v = fy y + oy
        gxx += -fx * (dJ0[0] * y - 2.f * x * dJ0[1] + dJ0[5] * iZ) - fy * (-dJ1[1] * y - dJ1[2]);
        gyy += -fx * (dJ0[0] * x + dJ0[2]) - fy * (2.f * y * dJ1[0] - dJ1[1] * x + dJ1[5] * iZ);
        giZ += -fx * (-dJ0[3] + dJ0[5] * x) - fy * (-dJ1[4] + dJ1[5] * y);
        grx = dj0 * fx * iZ; gry = dj1 * fy * iZ; grz = -dj0 * fx * x * iZ - dj1 * fy * y * iZ;
        gxx += -dj0 * fx * rz * iZ; gyy += -dj1 * fy * rz * iZ;
        giZ += dj0 * fx * (rx - rz * x) + dj1 * fy * (ry - rz * y);
        gX = gxx * iZ; gY = gyy * iZ; gZ = -iZ * (gxx * x + gyy * y) - iZ * iZ * giZ;
        gDt = rx * gX + ry * gY + rz * gZ;
        grx += Dt * gX; gry += Dt * gY; grz += Dt * gZ;
    }
};


// ---- reduction --------------------------------------------------------------------------------------------------------------------------
// The partial slots of group g (a pair, or a window; its tiles are [p0, p1)) of a build whose prm.total_tiles tiles were split contiguously
// over grid_build CTAs: one per CTA whose tile range intersects [p0, p1), a contiguous CTA range, at prm.partials + (cta prm.max_span +
// span) prm.slot_floats.  The first is found from c0 = floor(p0 grid / total), which is never past it (part_begin(c0) <= p0).  Writes
// them into s_slot (a pair can be spread over the whole grid, at most 2 CTAs per SM), returns their number.
constexpr int kMaxSlots = 2 * kMaxSMs + 8;
template <typename Params>
__device__ __forceinline__ int find_slots(const Params& prm, int grid_build, int tiles_per_group, int g, long long p0, long long p1, const float** s_slot) {
    int c0 = (int)((p0 * grid_build) / prm.total_tiles);
    while (c0 + 1 < grid_build && part_begin(prm.total_tiles, grid_build, c0 + 1) <= p0) ++c0;
    int n = 0;
    for (int c = c0; c < grid_build && n < kMaxSlots; ++c) {
        const long long tb = part_begin(prm.total_tiles, grid_build, c), te = part_begin(prm.total_tiles, grid_build, c + 1);
        if (tb >= p1) break;
        if (tb >= te || te <= p0) continue;
        const int span = g - (int)(tb / tiles_per_group);
        s_slot[n++] = prm.partials + ((size_t)c * prm.max_span + span) * prm.slot_floats;
    }
    return n;
}

}  // namespace banet
