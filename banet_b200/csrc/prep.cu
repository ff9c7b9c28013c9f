// Level pre-/post-steps: rays, grad_fixed(+concat,+half swap), bilinear resampler, depth composition.
// All are one-pass streaming kernels (HBM-bound, coalesced along the channel axis).
#include "common.cuh"
#include "features.cuh"
#include "lm_build.h"
#include "point.cuh"

namespace banet {

// BundleNet.computeCoordinates (reference bundlenet.py:112-120; legacy/ba.py:27-34 when !normalize)
__global__ void compute_coordinates_kernel(const float* __restrict__ points, const float* __restrict__ intr,
                                           int nb, int N, int normalize, float* __restrict__ p)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)nb * N) return;
    const int b = (int)(i / N), n = (int)(i - (long long)b * N);
    const float fx = intr[b * 4], fy = intr[b * 4 + 1], ox = intr[b * 4 + 2], oy = intr[b * 4 + 3];
    const float2 uv = reinterpret_cast<const float2*>(points)[i];
    float x = (uv.x - ox) / fx, y = (uv.y - oy) / fy, z = 1.f;
    if (normalize) {                                   // tf.nn.l2_normalize: x * rsqrt(max(sum sq, 1e-12))
        const float inv = 1.0f / sqrtf(fmaxf(x * x + y * y + 1.f, 1e-12f));
        x *= inv; y *= inv; z *= inv;
    }
    float* pb = p + (size_t)b * 3 * N;
    pb[n] = x; pb[(size_t)N + n] = y; pb[2 * (size_t)N + n] = z;
}

// grad_fixed + concat (+ half swap): bundlenet.py:92-100, 386-389.  One thread per (texel, 4 channels).
template <int VEC>
__global__ void grad_fixed_concat_kernel(const float* __restrict__ F, int nb, int h, int w, int C, int swap_halves,
                                         float* __restrict__ out)
{
    const int cv = C / VEC;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)nb * h * w * cv;
    if (i >= total) return;
    const int c = (int)(i % cv) * VEC;
    long long t = i / cv;
    const int x = (int)(t % w); t /= w;
    const int y = (int)(t % h); const int b = (int)(t / h);
    const int bs = swap_halves ? (b + nb / 2) % nb : b;            // layers[nb/2:nb] ++ layers[0:nb/2]
    const float* img = F + (size_t)bs * h * w * C;
    const int xe = reflect1(x + 1, w), xw = reflect1(x - 1, w), ys = reflect1(y + 1, h), yn = reflect1(y - 1, h);
    float* o = out + (((size_t)b * h + y) * w + x) * 3 * C;
#pragma unroll
    for (int u = 0; u < VEC; ++u) {
        const float f = img[((size_t)y * w + x) * C + c + u];
        const float gx = 0.5f * (img[((size_t)y * w + xe) * C + c + u] - img[((size_t)y * w + xw) * C + c + u]);
        const float gy = 0.5f * (img[((size_t)ys * w + x) * C + c + u] - img[((size_t)yn * w + x) * C + c + u]);
        o[c + u] = f; o[C + c + u] = gx; o[2 * C + c + u] = gy;
    }
}

// legacy/utils_python.py:61-117 `interpolate2d` / :177-232 `interpolate2d2`: bilinear with CLAMPED tap indices (:96-99) and, optionally, the
// in-bounds mask (x == clip(x, 0, w-1)) & (y == clip(y, 0, h-1)) (:114-116).  Warp per point, lanes over channels.
__global__ void interpolate2d_kernel(const float* __restrict__ data, const float* __restrict__ xy, float cs,
                                     int nb, int h, int w, int C, int N, float* __restrict__ out, float* __restrict__ mask)
{
    const long long pt = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (pt >= (long long)nb * N) return;
    const int b = (int)(pt / N);
    const float x = xy[pt * 2] * cs, y = xy[pt * 2 + 1] * cs;
    const float fx = floorf(x), fy = floorf(y);
    const float dx = x - fx, dy = y - fy;
    const bool fin = isfinite(x) && isfinite(y) && fabsf(x) < 1e9f && fabsf(y) < 1e9f;
    const int xi = fin ? (int)fx : 0, yi = fin ? (int)fy : 0;
    const int x0 = min(max(xi, 0), w - 1), x1 = min(max(xi + 1, 0), w - 1), y0 = min(max(yi, 0), h - 1), y1 = min(max(yi + 1, 0), h - 1);
    const float w00 = (1.f - dx) * (1.f - dy), w01 = dx * (1.f - dy), w10 = (1.f - dx) * dy, w11 = dx * dy;
    const float* img = data + (size_t)b * h * w * C;
    const float *t00 = img + ((size_t)y0 * w + x0) * C, *t01 = img + ((size_t)y0 * w + x1) * C, *t10 = img + ((size_t)y1 * w + x0) * C, *t11 = img + ((size_t)y1 * w + x1) * C;
    float* o = out + (size_t)pt * C;
    for (int c = lane; c < C; c += 32) o[c] = w00 * __ldg(t00 + c) + w01 * __ldg(t01 + c) + w10 * __ldg(t10 + c) + w11 * __ldg(t11 + c);
    if (mask && lane == 0) mask[pt] = (x >= 0.f && x <= (float)(w - 1) && y >= 0.f && y <= (float)(h - 1)) ? 1.f : 0.f;
}

// tf.contrib.resampler.resampler: bilinear, zero outside.  Warp per point, lanes over channels.  TF: float, or bf16 in and out (fp32
// arithmetic, rounded to nearest on store).
__device__ __forceinline__ void store_feat(float* p, float v) { *p = v; }
__device__ __forceinline__ void store_feat(bf16* p, float v) { *p = __float2bfloat16_rn(v); }
template <typename TF>
__global__ void resample_kernel(const TF* __restrict__ data, const float* __restrict__ xy, float cs,
                                int nb, int h, int w, int C, int N, TF* __restrict__ out)
{
    const long long pt = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (pt >= (long long)nb * N) return;
    const int b = (int)(pt / N);
    const float x = xy[pt * 2] * cs, y = xy[pt * 2 + 1] * cs;
    const float fx = floorf(x), fy = floorf(y);
    const float dx = x - fx, dy = y - fy;
    const bool fin = isfinite(x) && isfinite(y) && fabsf(x) < 1e9f && fabsf(y) < 1e9f;
    const int x0 = fin ? (int)fx : -10, y0 = fin ? (int)fy : -10;
    const float wt[4] = {(1.f - dx) * (1.f - dy), dx * (1.f - dy), (1.f - dx) * dy, dx * dy};
    const TF* img = data + (size_t)b * h * w * C;
    TF* o = out + (size_t)pt * C;
    for (int c = lane; c < C; c += 32) {
        float acc = 0.f;
#pragma unroll
        for (int tp = 0; tp < 4; ++tp) {
            const int xx = x0 + (tp & 1), yy = y0 + (tp >> 1);
            if (xx >= 0 && xx < w && yy >= 0 && yy < h) acc = fmaf(wt[tp], ldg_feat(img + ((size_t)yy * w + xx) * C + c), acc);
        }
        store_feat(o + c, acc);
    }
}

// bundlenet.py:397: depth = init_depth + basis . W.   Warp per output texel.  TB: basis element type (float, or bf16 widened on load).
template <typename TB>
__global__ void depth_compose_kernel(const float* __restrict__ init_depth, const TB* __restrict__ basis,
                                     const float* __restrict__ W, int nb, int M, int K, float* __restrict__ out)
{
    const long long pt = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (pt >= (long long)nb * M) return;
    const int b = (int)(pt / M);
    const TB* br = basis + (size_t)pt * K;
    const float* wb = W + (size_t)b * K;
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) acc = fmaf(ld_stream_elem(br + k), __ldg(wb + k), acc);
    acc = warp_sum(acc);
    if (lane == 0) out[pt] = init_depth[pt] + acc;
}

// Backward of grad_fixed + concat (+ half swap): dF[b'][y][x][c] = dconv2_F + 0.5 * sum of the gx / gy gradients of the texels whose
// REFLECT-by-one stencil reads (x,y) (transposed stencil; a border texel's neighbour is read twice, with opposite signs on the reflected
// side).  Gather form (no atomics): for texel x, the texels x' in {x-1, x+1} read it as their east / west neighbour, plus the reflected
// reads of the border columns.  One thread per (texel, channel).
__global__ void grad_fixed_concat_bwd_kernel(const float* __restrict__ dconv2, int nb, int h, int w, int C, int swap_halves, float* __restrict__ dF)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)nb * h * w * C;
    if (i >= total) return;
    const int c = (int)(i % C);
    long long t = i / C;
    const int x = (int)(t % w); t /= w;
    const int y = (int)(t % h); const int b = (int)(t / h);
    const float* g = dconv2 + (size_t)b * h * w * 3 * C;
    auto G = [&](int yy, int xx, int which) { return g[((size_t)yy * w + xx) * 3 * C + which * C + c]; };
    float acc = G(y, x, 0);
    // gx(x') = 0.5 (F[reflect(x'+1)] - F[reflect(x'-1)]):  x is the east neighbour of x' when reflect(x'+1) == x, the west one when reflect(x'-1) == x
    for (int xp = max(0, x - 1); xp <= min(w - 1, x + 1); ++xp) {
        if (reflect1(xp + 1, w) == x) acc += 0.5f * G(y, xp, 1);
        if (reflect1(xp - 1, w) == x) acc -= 0.5f * G(y, xp, 1);
    }
    for (int yp = max(0, y - 1); yp <= min(h - 1, y + 1); ++yp) {
        if (reflect1(yp + 1, h) == y) acc += 0.5f * G(yp, x, 2);
        if (reflect1(yp - 1, h) == y) acc -= 0.5f * G(yp, x, 2);
    }
    const int bs = swap_halves ? (b + nb / 2) % nb : b;            // forward: output pair b read input pair bs
    dF[(((size_t)bs * h + y) * w + x) * C + c] = acc;
}

// Backward of the resampler w.r.t. the sampled map: scatter (atomics).  Warp per point, lanes over channels.  dData must be zero-filled.
__global__ void resample_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ xy, float cs,
                                    int nb, int h, int w, int C, int N, float* __restrict__ ddata)
{
    const long long pt = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (pt >= (long long)nb * N) return;
    const int b = (int)(pt / N);
    const float x = xy[pt * 2] * cs, y = xy[pt * 2 + 1] * cs;
    const float fx = floorf(x), fy = floorf(y);
    const float dx = x - fx, dy = y - fy;
    const bool fin = isfinite(x) && isfinite(y) && fabsf(x) < 1e9f && fabsf(y) < 1e9f;
    const int x0 = fin ? (int)fx : -10, y0 = fin ? (int)fy : -10;
    const float wt[4] = {(1.f - dx) * (1.f - dy), dx * (1.f - dy), (1.f - dx) * dy, dx * dy};
    float* img = ddata + (size_t)b * h * w * C;
    const float* o = dout + (size_t)pt * C;
    for (int c = lane; c < C; c += 32) {
        const float gv = o[c];
#pragma unroll
        for (int tp = 0; tp < 4; ++tp) {
            const int xx = x0 + (tp & 1), yy = y0 + (tp >> 1);
            if (xx >= 0 && xx < w && yy >= 0 && yy < h) atomicAdd(img + ((size_t)yy * w + xx) * C + c, wt[tp] * gv);
        }
    }
}

// Backward of depth_compose: dinit = dout; dbasis[pt][k] = dout[pt] W[k]; dW[k] += sum_pt dout[pt] basis[pt][k] (atomics; dW zero-filled).
// One batch entry per blockIdx.y, striding by gridDim.y when nb exceeds the y dimension's limit.
template <typename TB>
__global__ void depth_compose_bwd_kernel(const float* __restrict__ dout, const TB* __restrict__ basis, const float* __restrict__ W,
                                         int nb, int M, int K, float* __restrict__ dbasis, float* __restrict__ dW)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    extern __shared__ float sacc[];              // [K]
    const int per = (M + gridDim.x - 1) / gridDim.x;
    const int m0 = blockIdx.x * per, m1 = min(M, m0 + per);
    for (int b = blockIdx.y; b < nb; b += gridDim.y) {
        for (int k = threadIdx.x; k < K; k += blockDim.x) sacc[k] = 0.f;
        __syncthreads();
        for (int k0 = 0; k0 < K; k0 += 32) {
            const int k = k0 + lane;
            const float wk = k < K ? W[(size_t)b * K + k] : 0.f;
            float acc = 0.f;
            for (int m = m0 + warp; m < m1; m += nw) {
                const size_t pt = (size_t)b * M + m;
                const float gv = dout[pt];
                if (k < K) {
                    float bv;
                    if constexpr (sizeof(TB) == 4) bv = basis[pt * K + k]; else bv = ldg_feat(basis + pt * K + k);
                    acc = fmaf(gv, bv, acc); dbasis[pt * K + k] = gv * wk;
                }
            }
            if (k < K) atomicAdd(&sacc[k], acc);
        }
        __syncthreads();
        for (int k = threadIdx.x; k < K; k += blockDim.x) atomicAdd(dW + (size_t)b * K + k, sacc[k]);
        __syncthreads();                         // sacc is cleared again for the next entry
    }
}

}  // namespace banet

using namespace banet;

extern "C" int banet_grad_fixed_concat_bwd(const float* dconv2, int nb, int h, int w, int C, int swap_halves, float* dF, banet_stream_t stream)
{
    BANET_REQUIRE(dconv2 && dF && nb > 0 && h >= 2 && w >= 2 && C > 0, BANET_ERR_BAD_ARG, "grad_fixed_concat_bwd: bad argument (need h,w >= 2)");
    BANET_REQUIRE(!swap_halves || nb % 2 == 0, BANET_ERR_BAD_ARG, "grad_fixed_concat_bwd: swap_halves needs an even batch");
    const long long tot = (long long)nb * h * w * C;
    grad_fixed_concat_bwd_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dconv2, nb, h, w, C, swap_halves, dF);
    BANET_CUDA_LAUNCH_CHECK("grad_fixed_concat_bwd");
    return BANET_OK;
}

extern "C" int banet_resample_bwd(const float* dout, const float* xy, float coord_scale, int nb, int h, int w, int C, int N,
                                  float* ddata, banet_stream_t stream)
{
    BANET_REQUIRE(dout && xy && ddata && nb > 0 && h > 0 && w > 0 && C > 0 && N > 0, BANET_ERR_BAD_ARG, "resample_bwd: bad argument");
    cudaMemsetAsync(ddata, 0, (size_t)nb * h * w * C * sizeof(float), (cudaStream_t)stream);
    const long long thr = (long long)nb * N * 32;
    resample_bwd_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dout, xy, coord_scale, nb, h, w, C, N, ddata);
    BANET_CUDA_LAUNCH_CHECK("resample_bwd");
    return BANET_OK;
}

namespace {
template <typename TB>
int depth_compose_bwd(const float* dout, const TB* basis, const float* W, int nb, int M, int K, float* dbasis, float* dW, cudaStream_t st,
                      const char* who)
{
    BANET_REQUIRE(dout && basis && W && dbasis && dW && nb > 0 && M > 0 && K > 0 && K <= 8192, BANET_ERR_BAD_ARG, "%s: bad argument", who);
    cudaMemsetAsync(dW, 0, (size_t)nb * K * sizeof(float), st);
    int gx = (M + 1023) / 1024; if (gx < 1) gx = 1; if (gx > 64) gx = 64;
    depth_compose_bwd_kernel<TB><<<dim3(gx, grid_y(nb)), 256, K * sizeof(float), st>>>(dout, basis, W, nb, M, K, dbasis, dW);
    BANET_CUDA_LAUNCH_CHECK(who);
    return BANET_OK;
}
template <typename TB>
int depth_compose(const float* init_depth, const TB* basis, const float* W, int nb, int M, int K, float* out, cudaStream_t st, const char* who)
{
    BANET_REQUIRE(init_depth && basis && W && out && nb > 0 && M > 0 && K > 0, BANET_ERR_BAD_ARG, "%s: bad argument", who);
    const long long thr = (long long)nb * M * 32;
    depth_compose_kernel<TB><<<(unsigned)((thr + 255) / 256), 256, 0, st>>>(init_depth, basis, W, nb, M, K, out);
    BANET_CUDA_LAUNCH_CHECK(who);
    return BANET_OK;
}
}  // namespace

extern "C" int banet_depth_compose_bwd(const float* dout, const float* basis, const float* W, int nb, int M, int K,
                                       float* dbasis, float* dW, banet_stream_t stream)
{
    return depth_compose_bwd(dout, basis, W, nb, M, K, dbasis, dW, (cudaStream_t)stream, "depth_compose_bwd");
}

extern "C" int banet_depth_compose_bwd_bf16(const float* dout, const void* basis, const float* W, int nb, int M, int K,
                                            float* dbasis, float* dW, banet_stream_t stream)
{
    return depth_compose_bwd(dout, static_cast<const bf16*>(basis), W, nb, M, K, dbasis, dW, (cudaStream_t)stream, "depth_compose_bwd_bf16");
}

extern "C" int banet_compute_coordinates(const float* points, const float* intr, int nb, int N, int normalize,
                                         float* p, banet_stream_t stream)
{
    BANET_REQUIRE(points && intr && p && nb > 0 && N > 0, BANET_ERR_BAD_ARG, "compute_coordinates: bad argument");
    const long long tot = (long long)nb * N;
    compute_coordinates_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, (cudaStream_t)stream>>>(points, intr, nb, N, normalize, p);
    BANET_CUDA_LAUNCH_CHECK("compute_coordinates");
    return BANET_OK;
}

extern "C" int banet_grad_fixed_concat(const float* F, int nb, int h, int w, int C, int swap_halves,
                                       float* conv2, banet_stream_t stream)
{
    BANET_REQUIRE(F && conv2 && nb > 0 && h >= 2 && w >= 2 && C > 0, BANET_ERR_BAD_ARG, "grad_fixed_concat: bad argument (need h,w >= 2)");
    BANET_REQUIRE(!swap_halves || nb % 2 == 0, BANET_ERR_BAD_ARG, "grad_fixed_concat: swap_halves needs an even batch");
    if (C % 4 == 0) {
        const long long tot = (long long)nb * h * w * (C / 4);
        grad_fixed_concat_kernel<4><<<(unsigned)((tot + 255) / 256), 256, 0, (cudaStream_t)stream>>>(F, nb, h, w, C, swap_halves, conv2);
    } else {
        const long long tot = (long long)nb * h * w * C;
        grad_fixed_concat_kernel<1><<<(unsigned)((tot + 255) / 256), 256, 0, (cudaStream_t)stream>>>(F, nb, h, w, C, swap_halves, conv2);
    }
    BANET_CUDA_LAUNCH_CHECK("grad_fixed_concat");
    return BANET_OK;
}

extern "C" int banet_resample(const float* data, const float* xy, float coord_scale, int nb, int h, int w, int C, int N,
                              float* out, banet_stream_t stream)
{
    BANET_REQUIRE(data && xy && out && nb > 0 && h > 0 && w > 0 && C > 0 && N > 0, BANET_ERR_BAD_ARG, "resample: bad argument");
    const long long thr = (long long)nb * N * 32;
    resample_kernel<float><<<(unsigned)((thr + 255) / 256), 256, 0, (cudaStream_t)stream>>>(data, xy, coord_scale, nb, h, w, C, N, out);
    BANET_CUDA_LAUNCH_CHECK("resample");
    return BANET_OK;
}

extern "C" int banet_resample_bf16(const void* data, const float* xy, float coord_scale, int nb, int h, int w, int C, int N,
                                   void* out, banet_stream_t stream)
{
    BANET_REQUIRE(data && xy && out && nb > 0 && h > 0 && w > 0 && C > 0 && N > 0, BANET_ERR_BAD_ARG, "resample_bf16: bad argument");
    const long long thr = (long long)nb * N * 32;
    resample_kernel<bf16><<<(unsigned)((thr + 255) / 256), 256, 0, (cudaStream_t)stream>>>(static_cast<const bf16*>(data), xy, coord_scale, nb, h, w,
                                                                                         C, N, static_cast<bf16*>(out));
    BANET_CUDA_LAUNCH_CHECK("resample_bf16");
    return BANET_OK;
}

extern "C" int banet_interpolate2d(const float* data, const float* xy, float coord_scale, int nb, int h, int w, int C, int N,
                                   float* out, float* mask, banet_stream_t stream)
{
    BANET_REQUIRE(data && xy && out && nb > 0 && h > 0 && w > 0 && C > 0 && N > 0, BANET_ERR_BAD_ARG, "interpolate2d: bad argument");
    const long long thr = (long long)nb * N * 32;
    interpolate2d_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, (cudaStream_t)stream>>>(data, xy, coord_scale, nb, h, w, C, N, out, mask);
    BANET_CUDA_LAUNCH_CHECK("interpolate2d");
    return BANET_OK;
}

extern "C" int banet_depth_compose(const float* init_depth, const float* basis, const float* W, int nb, int M, int K,
                                   float* out, banet_stream_t stream)
{
    return depth_compose(init_depth, basis, W, nb, M, K, out, (cudaStream_t)stream, "depth_compose");
}

extern "C" int banet_depth_compose_bf16(const float* init_depth, const void* basis, const float* W, int nb, int M, int K,
                                        float* out, banet_stream_t stream)
{
    return depth_compose(init_depth, static_cast<const bf16*>(basis), W, nb, M, K, out, (cudaStream_t)stream, "depth_compose_bf16");
}
