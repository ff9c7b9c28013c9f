// Shared helpers for the sm_90a kernels of libbanet.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/banet_abi.h"

namespace banet {

void set_error(const char* fmt, ...);

#define BANET_REQUIRE(cond, code, ...)                 \
    do { if (!(cond)) { ::banet::set_error(__VA_ARGS__); return (code); } } while (0)

#define BANET_CUDA_LAUNCH_CHECK(what)                                              \
    do { cudaError_t e__ = cudaGetLastError();                                     \
         if (e__ != cudaSuccess) { ::banet::set_error("%s: %s", what, cudaGetErrorString(e__)); \
                                   return BANET_ERR_CUDA; } } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

constexpr int kMaxSMs = 132;          // H100 SXM
constexpr int kMaxGridY = 65535;      // gridDim.y limit: launches with the batch on y stride over it (blockIdx.y, += gridDim.y)

static inline unsigned grid_y(long long n) { return (unsigned)(n < kMaxGridY ? n : kMaxGridY); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Robust loss of a point (banet_level_t::robust, robust_scale = delta) at s = |d|^2, the squared norm of its residual over the channels:
// rho'(s), the factor of its IRLS weight, and rho''(s) (d2, for the backward).  Every kernel that weighs points by a robust loss calls
// this one function.  BANET_ROBUST_NONE: rho(s) = s, rho' = 1 exactly, so a non-robust weight is multiplied by 1.0f.
//   Huber   rho(s) = s (s <= delta^2), 2 delta sqrt(s) - delta^2       rho' = 1 or delta / sqrt(s)      rho'' = 0 or -rho' / (2 s)
//   Cauchy  rho(s) = delta^2 log(1 + s / delta^2)                     rho' = delta^2 / (delta^2 + s)   rho'' = -delta^2 / (delta^2 + s)^2
__device__ __forceinline__ float robust_rho1(int kind, float delta, float s, float* d2 = nullptr)
{
    float r1 = 1.f, r2 = 0.f;
    if (kind == BANET_ROBUST_HUBER) {
        if (s > delta * delta) { r1 = delta / sqrtf(s); r2 = -0.5f * r1 / s; }
    } else if (kind == BANET_ROBUST_CAUCHY) {
        const float t = delta * delta, u = t + s;
        r1 = t / u; r2 = -r1 / u;
    }
    if (d2) *d2 = r2;
    return r1;
}
// rho(s) itself, the loss whose derivative robust_rho1 gives (the same branch at s = delta^2): the feature-metric cost of a point.
__device__ __forceinline__ float robust_rho(int kind, float delta, float s)
{
    if (kind == BANET_ROBUST_HUBER) {
        const float t = delta * delta;
        return s > t ? 2.f * delta * sqrtf(s) - t : s;
    }
    if (kind == BANET_ROBUST_CAUCHY) {
        const float t = delta * delta;
        return t * log1pf(s / t);
    }
    return s;
}

// streaming 128-bit load that does not pollute L1 (read-once data: conv1, B)
__device__ __forceinline__ float4 ld_stream_f4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ float ld_stream_f1(const float* p) {
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}

// Static contiguous partition of `total` work units over `parts` workers (deterministic).
__host__ __device__ __forceinline__ long long part_begin(long long total, int parts, int i) {
    return total * (long long)i / (long long)parts;
}

// ---- layout of one partial-sum slot written by the build kernel (floats) --------------------
//   [0, K*K)            Hdd   row-major full K x K
//   [K*K, K*K+7K)       ext   rows 0..5: H_cd[i][k] ; row 6: g_d[k]
//   then 32 floats      cc    21 upper-tri H_cc (row-major i<=j) + 6 g_c + nvalid + pad
//   then C floats       rbar partial sums
struct SlotLayout {
    int K, C;
    __host__ __device__ int off_ext()  const { return K * K; }
    __host__ __device__ int off_cc()   const { return K * K + 7 * K; }
    __host__ __device__ int off_rbar() const { return K * K + 7 * K + 32; }
    __host__ __device__ int floats()   const { return ((K * K + 7 * K + 32 + C) + 3) / 4 * 4; }
};

}  // namespace banet
