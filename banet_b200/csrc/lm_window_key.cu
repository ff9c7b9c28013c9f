// lm_window_key.cu — normal equations of keyframe windows whose keyframe tensors are given once per window (ABI section 3e), and their
// backward.  fp32 SIMT, the arithmetic of lm_build_kernel / lm_build_bwd_kernel.
//
// Window w holds nf pairs (keyframe of w -> frame f), pair w nf + f.  Every pair samples the same keyframe points with the same depth
// D + B.W_w, so the per-pair depth blocks and couplings share the basis:
//     sum_f H_dd,f = B^T diag(sum_f s_f) B          [H_cd,f | g_d,f]^T = B^T [v_f | t_f]      (s_f = jd^T M_f jd, v_f, t_f per point)
// and one contraction of B against K + 7 nf columns gives them all (the per-pair build contracts nf times against K + 7).
//
// Output: the "window-reduced" per-pair system.  H [nw nf,P,P], g, rbar_sum, nvalid are the per-pair values of banet_lm_build except that
// frame 0's depth block holds the window's whole depth block sum_f H_dd,f and every other frame's depth block is exactly zero.  The window
// steps (banet_lm_window_batch_solve_update, banet_lm_window_solve_update) only ever sum the depth blocks over the frames, so they take this
// layout as it is.
//
// keyframe_build_kernel: the nw ceil(N/64) point tiles are split contiguously over a persistent grid (as lm_build_kernel does with pairs).
// Per tile: stage the basis rows and D + b.W_w once, walk the frames in order (geometry, gather, per-point records), contract the tile's
// [v_f | t_f] columns of each frame against B, then contract B against diag(sum_f s_f) B.  The H_dd accumulators stay in registers across
// the tiles of a window span; the per-frame H_cd, g_d, H_cc, g_c, nvalid and rbar sums go straight into the CTA's own partial slot (the
// first tile of a span stores, the others add: every element has one owner thread, no atomics).  keyframe_reduce_kernel sums the slots of a
// window in a fixed order in fp64.  Bit-reproducible; the workspace's previous contents are never read.
//
// keyframe_build_bwd_kernel: warp per point, the frames walked in order inside the point.  The basis row, D + b.W and e = b^T S_dd (the only
// K^2 term, with S_dd from frame 0's depth block of dH) are formed once per point; dconv1, dD, dB are summed over the frames and stored
// once, without atomics (bit-reproducible).  dconv2, dR, dT (per pair) and dW (per window) are accumulated with atomics as in lm_bwd.cu.
// The depth blocks of the other frames of dH are ignored: they are constants (zero) in the forward, so this is the exact adjoint.
//
// Point weights (banet_keyframe_level_t::weight, one per (frame, point), pair w nf + f): the forward scales a point's M, q in each frame after
// its channel reduction, so every weighted quantity (H_cc, g_c, v_f, t_f, s_f and with s_f the window's depth block) follows; sum |d| and
// nvalid stay unweighted.  The backward stores dw = 1/2 <M, Q> + q.z per (frame, point) and scales that point's adjoints by w.
//
// The per-point code (geometry, gather, Jacobians, the chain rule through the sampler) is point.cuh's, shared with lm_build_kernel and
// lm_build_bwd_kernel; this file holds what differs for a keyframe given once: the tile and frame loops, the slot layout and the commits.
#include "common.cuh"
#include "lm_build.h"
#include "point.cuh"

namespace banet {
namespace {

constexpr int KT_PX = 64;                    // points per tile
constexpr int KT_THREADS = 256;
constexpr int KT_WARPS = KT_THREADS / 32;

enum { R_X0 = 0, R_Y0, R_DX, R_DY, R_MASK, R_X, R_Y, R_IZ, R_RX, R_RY, R_RZ, R_M11, R_M12, R_M22, R_Q1, R_Q2, R_P0, R_P1, R_P2, R_DT, R_SSUM, R_ANY,
       KT_REC };

// partial slot (floats): H_dd [K][K] | per frame f at frame_off(f): ext [7][K] (H_cd rows 0..5, g_d row 6) | cc [32] (21 H_cc, 6 g_c, nvalid) | rbar [C]
struct KeySlot {
    int K, C;
    __host__ __device__ int frame_floats() const { return (7 * K + 32 + C + 3) / 4 * 4; }
    __host__ __device__ size_t frame_off(int f) const { return (size_t)K * K + (size_t)f * frame_floats(); }
    __host__ __device__ size_t floats(int nf) const { return frame_off(nf); }
};

struct KeyParams {
    int nw, nf, N, C, K, h, w, c2;
    const float *conv1, *p, *D, *B;          // keyframe, [nw,...]
    const float *conv2, *intr, *R, *T;       // per pair, [nw nf,...]
    const float* W;                          // [nw,K]
    const float* weight;                     // [nw nf,N] point weights per pair, or NULL (= 1)
    float* partials;
    size_t slot_floats;
    int max_span, tiles_per_win;
    long long total_tiles;
    int kq_i, kq_j;                          // K > 128: the 128 x 128 block of H_dd this launch computes
};

template <int KP> struct KeySmem {
    static constexpr int LDB = KP + 4;
    static constexpr int off_B = 0;
    static constexpr int off_W = off_B + KT_PX * LDB;
    static constexpr int off_rec = off_W + KP;
    static constexpr int off_ext = off_rec + KT_REC * KT_PX;            // [KT_PX][8]: v0..v5, t, s of the current frame
    static constexpr int off_pose = off_ext + KT_PX * 8;                // R(9) T(3) intr(4)
    static constexpr int off_cc = off_pose + 16;                        // [2][32]
    static constexpr int off_rb = off_cc + 64;                          // [KT_WARPS][C]
    static size_t bytes(int C) { return (size_t)(off_rb + KT_WARPS * C) * sizeof(float); }
};

template <int KP, int VEC>
__global__ void __launch_bounds__(KT_THREADS, (KP >= 128) ? 1 : 2)
keyframe_build_kernel(const KeyParams prm)
{
    using SM = KeySmem<KP>;
    extern __shared__ __align__(16) float smem[];
    float* Bs = smem + SM::off_B;
    float* sW = smem + SM::off_W;
    float* rec = smem + SM::off_rec;
    float* sExt = smem + SM::off_ext;
    float* sPose = smem + SM::off_pose;
    float* sCC = smem + SM::off_cc;
    float* sRb = smem + SM::off_rb;
    constexpr int LDB = SM::LDB;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = prm.N, C = prm.C, K = prm.K, h = prm.h, w = prm.w, c2 = prm.c2, nf = prm.nf;
    const bool fly = (c2 == C);

    // register tile of H_dd as in lm_build_kernel (K > 128: one 128 x 128 block of its lower triangle per launch)
    constexpr int KB = (KP > 128) ? 128 : KP;
    const int ki0 = (KP > 128) ? prm.kq_i * 128 : 0, kj0 = (KP > 128) ? prm.kq_j * 128 : 0;
    const bool first_block = (KP <= 128) || (prm.kq_i == 0 && prm.kq_j == 0), diag_block = (KP <= 128) || (prm.kq_i == prm.kq_j);
    constexpr int T = KB / 16;
    constexpr int G = (T >= 4) ? 4 : T;
    constexpr int NG = T / G;
    constexpr int NPART = KT_THREADS / KB;
    constexpr int EA = (7 + NPART - 1) / NPART;
    float acc[T][T];
    const int ti = tid >> 4, tj = tid & 15;
    const KeySlot L{K, C};

    const long long t_begin = part_begin(prm.total_tiles, gridDim.x, blockIdx.x);
    const long long t_end = part_begin(prm.total_tiles, gridDim.x, blockIdx.x + 1);
    int cur_w = -1, span = 0;
    float* slot = nullptr;

    auto flush_hdd = [&]() {
#pragma unroll
        for (int e = 0; e < T; ++e) {
            const int row = ki0 + (e / G) * (16 * G) + G * ti + (e % G);
#pragma unroll
            for (int f = 0; f < T; ++f) {
                const int col = kj0 + (f / G) * (16 * G) + G * tj + (f % G);
                if (row < K && col < K) slot[row * K + col] = acc[e][f];
            }
        }
    };

    for (long long t = t_begin; t < t_end; ++t) {
        const int wi = (int)(t / prm.tiles_per_win);
        const int n0 = (int)(t - (long long)wi * prm.tiles_per_win) * KT_PX;
        const int cnt = min(KT_PX, N - n0);
        const bool first_tile = (wi != cur_w);            // first tile of this CTA's span of window wi: the slot is stored, not added to
        if (first_tile) {
            if (cur_w >= 0) { flush_hdd(); ++span; }
#pragma unroll
            for (int e = 0; e < T; ++e)
#pragma unroll
                for (int f = 0; f < T; ++f) acc[e][f] = 0.f;
            slot = prm.partials + ((size_t)blockIdx.x * prm.max_span + span) * prm.slot_floats;
            __syncthreads();                                 // the previous tile's readers of sW are done
            for (int k = tid; k < KP; k += KT_THREADS) sW[k] = (k < K) ? prm.W[(size_t)wi * K + k] : 0.f;
            cur_w = wi;
        }

        // ---- basis tile (coalesced, read once) -------------------------------------------------------------------------------
        const float* Bg = prm.B + ((size_t)wi * N + n0) * K;
        if ((K & 3) == 0) {
            const int k4 = K >> 2, kp4 = KP >> 2;
            for (int i = tid; i < KT_PX * kp4; i += KT_THREADS) {
                const int n = i / kp4, q = i - n * kp4;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (n < cnt && q < k4) v = ld_stream_f4(Bg + (size_t)n * K + 4 * q);
                *reinterpret_cast<float4*>(Bs + n * LDB + 4 * q) = v;
            }
        } else {
            for (int i = tid; i < KT_PX * KP; i += KT_THREADS) {
                const int n = i / KP, k = i - n * KP;
                Bs[n * LDB + k] = (n < cnt && k < K) ? ld_stream_f1(Bg + (size_t)n * K + k) : 0.f;
            }
        }
        __syncthreads();
        // ---- the keyframe's depth D + b.W_w and ray p, once per point --------------------------------------------------------
        if (tid < KT_PX) {
            const int n = tid;
            float p0 = 0.f, p1 = 0.f, p2 = 0.f, Dt = 0.f;
            if (n < cnt) {
                const float* pp = prm.p + (size_t)wi * 3 * N + n0 + n;
                p0 = pp[0]; p1 = pp[N]; p2 = pp[2 * (size_t)N];
                Dt = prm.D[(size_t)wi * N + n0 + n];
                Dt += basis_dot<KP>(Bs + n * LDB, sW);
            }
            rec[R_P0 * KT_PX + n] = p0; rec[R_P1 * KT_PX + n] = p1; rec[R_P2 * KT_PX + n] = p2; rec[R_DT * KT_PX + n] = Dt;
            rec[R_SSUM * KT_PX + n] = 0.f; rec[R_ANY * KT_PX + n] = 0.f;
        }

        // ---- the frames, in order ------------------------------------------------------------------------------------------------
        for (int f = 0; f < nf; ++f) {
            const int b = wi * nf + f;
            float* fslot = slot + L.frame_off(f);
            __syncthreads();                                 // previous frame's readers of the pose, records, sExt, sCC, sRb are done
            if (tid < 9) sPose[tid] = prm.R[b * 9 + tid];
            else if (tid < 12) sPose[tid] = prm.T[b * 3 + tid - 9];
            else if (tid < 16) sPose[tid] = prm.intr[b * 4 + tid - 12];
            for (int c = tid; c < KT_WARPS * C; c += KT_THREADS) sRb[c] = 0.f;
            __syncthreads();
            // S1: geometry, thread per point (bundlenet.py:208-224, mask :231)
            if (tid < KT_PX) {
                const int n = tid;
                float mask = 0.f, x = 0.f, y = 0.f, iZ = 0.f, rx = 0.f, ry = 0.f, rz = 0.f, dx = 0.f, dy = 0.f;
                int x0 = 0, y0 = 0;
                if (n < cnt) {
                    const float p0 = rec[R_P0 * KT_PX + n], p1 = rec[R_P1 * KT_PX + n], p2 = rec[R_P2 * KT_PX + n], Dt = rec[R_DT * KT_PX + n];
                    const Projection pr(sPose, p0, p1, p2, Dt);
                    rx = pr.rx; ry = pr.ry; rz = pr.rz; x = pr.x; y = pr.y; iZ = pr.iZ;
                    if (pr.in_bounds(h, w)) {
                        mask = 1.f;
                        tap_corner(pr.u, pr.v, x0, y0, dx, dy);
                    }
                }
                rec[R_X0 * KT_PX + n] = __int_as_float(x0); rec[R_Y0 * KT_PX + n] = __int_as_float(y0);
                rec[R_DX * KT_PX + n] = dx; rec[R_DY * KT_PX + n] = dy; rec[R_MASK * KT_PX + n] = mask;
                rec[R_X * KT_PX + n] = x; rec[R_Y * KT_PX + n] = y; rec[R_IZ * KT_PX + n] = iZ;
                rec[R_RX * KT_PX + n] = rx; rec[R_RY * KT_PX + n] = ry; rec[R_RZ * KT_PX + n] = rz;
            }
            __syncthreads();
            // S2: feature gather, warp per point, lanes over channels (bundlenet.py:230-239)
            for (int i = 0; i < KT_PX / KT_WARPS; ++i) {
                const int n = i * KT_WARPS + warp;
                PointMQ mq{0.f, 0.f, 0.f, 0.f, 0.f};
                const bool valid = rec[R_MASK * KT_PX + n] != 0.f;
                if (valid) {
                    const Taps tp(__float_as_int(rec[R_X0 * KT_PX + n]), __float_as_int(rec[R_Y0 * KT_PX + n]), rec[R_DX * KT_PX + n], rec[R_DY * KT_PX + n], h, w);
                    const TapGather<float> tg(prm.conv2 + (size_t)b * h * w * c2, tp, h, w, C, c2);
                    const float* c1 = prm.conv1 + ((size_t)wi * N + n0 + n) * C;      // the keyframe's features, re-read by every frame (L1 / L2)
                    float* myRb = sRb + warp * C;
                    for (int c = lane * VEC; c < C; c += 32 * VEC) {
                        ChanVec<VEC> f1;
                        f1.load(c1 + c);
                        tg.group<VEC>(f1, fly, c, myRb, mq);
                    }
                    mq.m11 = warp_sum(mq.m11); mq.m12 = warp_sum(mq.m12); mq.m22 = warp_sum(mq.m22); mq.q1 = warp_sum(mq.q1); mq.q2 = warp_sum(mq.q2);
                }
                if (lane == 0) {
                    // point weight of (frame f, point n): scales M and q, and through them every weighted quantity of S3 (H_cc, g_c, v_f,
                    // t_f, s_f); sum |d|, nvalid and R_ANY stay unweighted.  Unweighted: x * 1.0f is exact
                    const float wn = (prm.weight && valid) ? __ldg(prm.weight + (size_t)b * N + n0 + n) : 1.f;
                    rec[R_M11 * KT_PX + n] = mq.m11 * wn; rec[R_M12 * KT_PX + n] = mq.m12 * wn; rec[R_M22 * KT_PX + n] = mq.m22 * wn;
                    rec[R_Q1 * KT_PX + n] = mq.q1 * wn; rec[R_Q2 * KT_PX + n] = mq.q2 * wn;
                }
            }
            __syncthreads();
            // S3: per-point 2 x (6+1) algebra, thread per point (bundlenet.py:49-74); the 28 pose sums of the tile through the two warps
            if (tid < KT_PX) {
                const int n = tid;
                float ext[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                float cc[28];
#pragma unroll
                for (int q = 0; q < 28; ++q) cc[q] = 0.f;
                if (rec[R_MASK * KT_PX + n] != 0.f) {
                    const float x = rec[R_X * KT_PX + n], y = rec[R_Y * KT_PX + n], iZ = rec[R_IZ * KT_PX + n];
                    const PointMQ mq{rec[R_M11 * KT_PX + n], rec[R_M12 * KT_PX + n], rec[R_M22 * KT_PX + n], rec[R_Q1 * KT_PX + n], rec[R_Q2 * KT_PX + n]};
                    const float fx = sPose[12], fy = sPose[13];
                    float a0[6], a1[6], jd0, jd1;
                    camera_jacobian(fx, fy, x, y, iZ, a0, a1);
                    pose_terms(a0, a1, mq, cc);
                    cc[27] = 1.f;
                    depth_jacobian(fx, fy, rec[R_RX * KT_PX + n], rec[R_RY * KT_PX + n], rec[R_RZ * KT_PX + n], x, y, iZ, jd0, jd1);
                    depth_terms(a0, a1, jd0, jd1, mq, ext);
                    rec[R_SSUM * KT_PX + n] += ext[7];
                    rec[R_ANY * KT_PX + n] = 1.f;
                }
                *reinterpret_cast<float4*>(sExt + n * 8) = make_float4(ext[0], ext[1], ext[2], ext[3]);
                *reinterpret_cast<float4*>(sExt + n * 8 + 4) = make_float4(ext[4], ext[5], ext[6], ext[7]);
                if (first_block) {
#pragma unroll
                    for (int q = 0; q < 28; ++q) { const float v = warp_sum(cc[q]); if (lane == 0) sCC[warp * 32 + q] = v; }
                }
            }
            __syncthreads();
            // S4: this frame's couplings  [H_cd,f; g_d,f] += [v_f; t_f] b^T  over the tile, then into the slot
            if (diag_block) {
                const int k = kj0 + tid % KB, part = tid / KB;
                float ax[EA];
#pragma unroll
                for (int q = 0; q < EA; ++q) ax[q] = 0.f;
                for (int n = 0; n < cnt; ++n) {
                    if (rec[R_MASK * KT_PX + n] == 0.f) continue;
                    const float bk = Bs[n * LDB + k];
#pragma unroll
                    for (int q = 0; q < EA; ++q) {
                        const int r = part * EA + q;
                        if (r < 7) ax[q] = fmaf(sExt[n * 8 + r], bk, ax[q]);
                    }
                }
                if (k < K) {
#pragma unroll
                    for (int q = 0; q < EA; ++q) {
                        const int r = part * EA + q;
                        if (r < 7) { float* d = fslot + r * K + k; *d = first_tile ? ax[q] : *d + ax[q]; }
                    }
                }
            }
            if (first_block) {
                float* dcc = fslot + 7 * K;
                if (tid < 28) { const float v = sCC[tid] + sCC[32 + tid]; dcc[tid] = first_tile ? v : dcc[tid] + v; }
                float* drb = dcc + 32;
                for (int c = tid; c < C; c += KT_THREADS) {
                    float s = 0.f;
#pragma unroll
                    for (int wq = 0; wq < KT_WARPS; ++wq) s += sRb[wq * C + c];
                    drb[c] = first_tile ? s : drb[c] + s;
                }
            }
        }
        __syncthreads();
        // ---- S5: the window's depth block  H_dd += (sum_f s_f) b b^T  (fp32 FFMA, once per point) ------------------------------
#pragma unroll 2
        for (int n = 0; n < cnt; ++n) {
            if (rec[R_ANY * KT_PX + n] == 0.f) continue;
            const float s = rec[R_SSUM * KT_PX + n];
            float a[T], cv[T];
#pragma unroll
            for (int gq = 0; gq < NG; ++gq) {
                lds_group<G>(Bs + n * LDB + ki0 + gq * 16 * G + G * ti, a + gq * G);
                lds_group<G>(Bs + n * LDB + kj0 + gq * 16 * G + G * tj, cv + gq * G);
            }
#pragma unroll
            for (int e = 0; e < T; ++e) {
                const float sa = s * a[e];
#pragma unroll
                for (int f = 0; f < T; ++f) acc[e][f] = fmaf(sa, cv[f], acc[e][f]);
            }
        }
        __syncthreads();
    }
    if (cur_w >= 0) flush_hdd();
}

// ---- fixed-order fp64 reduction of the slots of each window -> the window-reduced per-pair system ----------------------------------
__device__ __forceinline__ void keyframe_reduce_window(const KeyParams& prm, int grid_build, int wi, float* __restrict__ H, float* __restrict__ g,
                                                       float* __restrict__ rbar_sum, float* __restrict__ nvalid)
{
    const int K = prm.K, C = prm.C, nf = prm.nf, P = 6 + K;
    const KeySlot L{K, C};
    const long long p0 = (long long)wi * prm.tiles_per_win, p1 = p0 + prm.tiles_per_win;
    __shared__ const float* s_slot[kMaxSlots];
    __shared__ int s_n;
    if (threadIdx.x == 0) s_n = find_slots(prm, grid_build, prm.tiles_per_win, wi, p0, p1, s_slot);
    __syncthreads();
    const int nslot = s_n;
    const int FF = 7 * K + 28 + C;                                    // used floats of a frame's part of the slot
    const long long nel = (long long)K * K + (long long)nf * FF;
    const size_t pair0 = (size_t)wi * nf;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nel; i += (long long)gridDim.x * blockDim.x) {
        if (i < (long long)K * K) {                                   // the window's depth block -> frame 0; the other frames get zeros
            const int r = (int)(i / K), cI = (int)(i - (long long)r * K);
            if (cI > r) continue;
            double s = 0.0;
            for (int q = 0; q < nslot; ++q) s += (double)s_slot[q][i];
            const float v = (float)s;
            H[(pair0 * P + 6 + r) * P + 6 + cI] = v; H[(pair0 * P + 6 + cI) * P + 6 + r] = v;
            for (int f = 1; f < nf; ++f) {
                const size_t b = pair0 + f;
                H[(b * P + 6 + r) * P + 6 + cI] = 0.f; H[(b * P + 6 + cI) * P + 6 + r] = 0.f;
            }
            continue;
        }
        const long long j = i - (long long)K * K;
        const int f = (int)(j / FF), e = (int)(j - (long long)f * FF);
        int src = e;                                                  // offset inside the frame's part of the slot (cc is padded to 32)
        if (e >= 7 * K + 28) src = e + 4;
        const size_t off = L.frame_off(f) + src;
        double s = 0.0;
        for (int q = 0; q < nslot; ++q) s += (double)s_slot[q][off];
        const float v = (float)s;
        const size_t b = pair0 + f;
        if (e < 7 * K) {
            const int rr = e / K, k = e - rr * K;
            if (rr < 6) { H[(b * P + rr) * P + 6 + k] = v; H[(b * P + 6 + k) * P + rr] = v; }
            else g[b * P + 6 + k] = v;
        } else if (e < 7 * K + 28) {
            const int q = e - 7 * K;
            if (q < 21) {
                int rr = 0, rem = q;
                while (rem >= 6 - rr) { rem -= 6 - rr; ++rr; }
                const int cc = rr + rem;
                H[(b * P + rr) * P + cc] = v; H[(b * P + cc) * P + rr] = v;
            } else if (q < 27) g[b * P + q - 21] = v;
            else nvalid[b] = v;
        } else {
            rbar_sum[b * C + (e - 7 * K - 28)] = v;
        }
    }
}

// One window per blockIdx.y, striding by gridDim.y when there are more windows than the y dimension allows.  Each element keeps its one
// summation order over the window's slots, so the result does not depend on the stride.
__global__ void __launch_bounds__(256)
keyframe_reduce_kernel(const KeyParams prm, int grid_build, float* __restrict__ H, float* __restrict__ g, float* __restrict__ rbar_sum,
                       float* __restrict__ nvalid)
{
    for (int wi = blockIdx.y; wi < prm.nw; wi += gridDim.y) {
        keyframe_reduce_window(prm, grid_build, wi, H, g, rbar_sum, nvalid);
        __syncthreads();                                              // every thread is done with this window's slot list
    }
}

template <int KP, int VEC>
int launch_key_build(const KeyParams& prm, int grid, cudaStream_t st)
{
    const size_t smem = KeySmem<KP>::bytes(prm.C);
    auto kern = keyframe_build_kernel<KP, VEC>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("keyframe_build: smem attr (%zu B): %s", smem, cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    kern<<<grid, KT_THREADS, smem, st>>>(prm);
    BANET_CUDA_LAUNCH_CHECK("keyframe_build_kernel launch");
    return BANET_OK;
}

// ------------------------------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------------------------------
constexpr int KB_THREADS = 512;
constexpr int KB_WARPS = KB_THREADS / 32;
constexpr int KB_TILE = 64;

struct KeyBwdParams {
    int nw, nf, N, C, K, h, w;
    const float *conv1, *p, *D, *B, *conv2, *intr, *R, *T, *W;
    const float *dH, *dg, *drbar;
    float *dconv1, *dconv2, *dD, *dB, *dR, *dT, *dW;
    const float* weight;                         // [nw nf,N] point weights per pair, or NULL (= 1)
    float* dweight;                              // [nw nf,N] their gradient, or NULL
    int exact_sym, nfc, tiles_per_win;
    long long total_tiles;
};

// shared memory (floats): S_dd [K][K] | W [K] | dconv1 row per warp [KB_WARPS][C] | per frame of the chunk (nfc of them, stride key_bwd_frame_floats):
//   S_cd [6][K] | S_dc [K][6] | S_cc [36] | ghat [P] | pose [16] | rhat [C] | dR, dT per warp [KB_WARPS][12]
__host__ __device__ inline size_t key_bwd_frame_floats(int K, int C) { return (size_t)12 * K + 36 + (6 + K) + 16 + C + KB_WARPS * 12; }
__host__ __device__ inline size_t key_bwd_fixed_floats(int K, int C) { return (size_t)K * K + K + (size_t)KB_WARPS * C; }

template <int KL>
__global__ void __launch_bounds__(KB_THREADS, 1)
keyframe_build_bwd_kernel(const KeyBwdParams prm)
{
    extern __shared__ __align__(16) float sm[];
    const int K = prm.K, C = prm.C, N = prm.N, h = prm.h, w = prm.w, P = 6 + K, C3 = 3 * C, nf = prm.nf;
    float* Sdd = sm;
    float* sW = Sdd + (size_t)K * K;
    float* sDc1 = sW + K;
    float* sFr = sDc1 + (size_t)KB_WARPS * C;
    const size_t FS = key_bwd_frame_floats(K, C);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float* myDc1 = sDc1 + (size_t)warp * C;
    const long long t_begin = part_begin(prm.total_tiles, gridDim.x, blockIdx.x);
    const long long t_end = part_begin(prm.total_tiles, gridDim.x, blockIdx.x + 1);

    for (long long ts = t_begin; ts < t_end;) {
        const int wi = (int)(ts / prm.tiles_per_win);
        const long long te = min(t_end, (long long)(wi + 1) * prm.tiles_per_win);
        __syncthreads();
        {   // S_dd from frame 0's depth block of dH (the other frames' depth blocks are constants of the forward)
            const float* Gh = prm.dH + (size_t)wi * nf * P * P;
            for (int i = tid; i < K * K; i += KB_THREADS) {
                const int r = i / K, c = i - r * K;
                const float a = Gh[(size_t)(6 + r) * P + 6 + c];
                Sdd[i] = prm.exact_sym ? (a + Gh[(size_t)(6 + c) * P + 6 + r]) : 2.f * a;
            }
            for (int i = tid; i < K; i += KB_THREADS) sW[i] = prm.W[(size_t)wi * K + i];
        }
        float accW[KL];
#pragma unroll
        for (int i = 0; i < KL; ++i) accW[i] = 0.f;

        for (int fc0 = 0; fc0 < nf; fc0 += prm.nfc) {
            const int nfl = min(prm.nfc, nf - fc0);
            __syncthreads();
            for (int fl = 0; fl < nfl; ++fl) {                        // this chunk's per-frame S_cc, S_cd, S_dc, ghat, pose, rhat
                const size_t b = (size_t)wi * nf + fc0 + fl;
                float* Fr = sFr + fl * FS;
                float *Scd = Fr, *Sdc = Scd + 6 * K, *Scc = Sdc + 6 * K, *sg = Scc + 36, *sPose = sg + P, *sRh = sPose + 16, *sRT = sRh + C;
                const float* Gh = prm.dH + b * P * P;
                for (int i = tid; i < 6 * P + 6 * K; i += KB_THREADS) {
                    int r, c;
                    if (i < 6 * P) { r = i / P; c = i - r * P; }         // rows 0..5: S_cc, S_cd
                    else { const int j = i - 6 * P; r = 6 + j / 6; c = j % 6; }   // rows 6..P-1, columns 0..5: S_dc
                    const float v = prm.exact_sym ? (Gh[(size_t)r * P + c] + Gh[(size_t)c * P + r]) : 2.f * Gh[(size_t)r * P + c];
                    if (r < 6 && c < 6) Scc[r * 6 + c] = v;
                    else if (r < 6) Scd[r * K + (c - 6)] = v;
                    else Sdc[(r - 6) * 6 + c] = v;
                }
                for (int i = tid; i < P; i += KB_THREADS) sg[i] = prm.dg[b * P + i];
                for (int i = tid; i < C; i += KB_THREADS) sRh[i] = prm.drbar[b * C + i];
                for (int i = tid; i < KB_WARPS * 12; i += KB_THREADS) sRT[i] = 0.f;
                if (tid < 9) sPose[tid] = prm.R[b * 9 + tid];
                else if (tid < 12) sPose[tid] = prm.T[b * 3 + tid - 9];
                else if (tid < 16) sPose[tid] = prm.intr[b * 4 + tid - 12];
            }
            __syncthreads();
            for (long long t = ts; t < te; ++t) {
                const int n0 = (int)(t - (long long)wi * prm.tiles_per_win) * KB_TILE;
                const int cnt = min(KB_TILE, N - n0);
                for (int pi = warp; pi < cnt; pi += KB_WARPS) {
                    const int n = n0 + pi;
                    const size_t gi = (size_t)wi * N + n;
                    // ---- once per point: basis row, depth, e = b^T S_dd, gamma = e.b -------------------------------------------------
                    float bl[KL], e[KL], db[KL];
                    float bw = 0.f;
#pragma unroll
                    for (int i = 0; i < KL; ++i) {
                        const int k = lane + 32 * i;
                        bl[i] = (k < K) ? ld_stream_f1(prm.B + gi * K + k) : 0.f;
                        if (k < K) bw = fmaf(bl[i], sW[k], bw);
                        e[i] = 0.f;
                        db[i] = (fc0 > 0 && k < K) ? prm.dB[gi * K + k] : 0.f;
                    }
                    bw = warp_sum(bw);
                    const float* pp = prm.p + (size_t)wi * 3 * N + n;
                    const float p0 = __ldg(pp), p1 = __ldg(pp + N), p2 = __ldg(pp + 2 * (size_t)N);
                    const float Dt = __ldg(prm.D + gi) + bw;                                 // bundlenet.py:208
#pragma unroll
                    for (int i2 = 0; i2 < KL; ++i2) {
                        if (32 * i2 >= K) break;
#pragma unroll 2
                        for (int j2 = 0; j2 < 32; ++j2) {
                            const int j = 32 * i2 + j2;
                            if (j >= K) break;
                            const float bj = __shfl_sync(0xffffffffu, bl[i2], j2);
                            const float* row = Sdd + (size_t)j * K;
#pragma unroll
                            for (int i = 0; i < KL; ++i) { const int k = lane + 32 * i; if (k < K) e[i] = fmaf(bj, row[k], e[i]); }
                        }
                    }
                    float gamma = 0.f;
#pragma unroll
                    for (int i = 0; i < KL; ++i) gamma = fmaf(e[i], bl[i], gamma);
                    gamma = warp_sum(gamma);
                    float dDacc = (fc0 > 0) ? prm.dD[gi] : 0.f;
                    const float* c1 = prm.conv1 + gi * C;
                    float* dc1 = prm.dconv1 + gi * C;
                    for (int c = lane; c < C; c += 32) myDc1[c] = (fc0 > 0) ? dc1[c] : 0.f;
                    __syncwarp();

                    for (int fl = 0; fl < nfl; ++fl) {
                        const size_t b = (size_t)wi * nf + fc0 + fl;
                        float* Fr = sFr + fl * FS;
                        const float *Scd = Fr, *Sdc = Scd + 6 * K, *Scc = Sdc + 6 * K, *sg = Scc + 36, *sPose = sg + P, *sRh = sPose + 16;
                        float* sRT = Fr + 13 * K + 58 + C + warp * 12;
                        const float fx = sPose[12], fy = sPose[13];
                        const Projection pr(sPose, p0, p1, p2, Dt);
                        if (!pr.in_bounds(h, w)) {                           // masked in this frame: no gradient through it
                            if (prm.dweight && lane == 0) prm.dweight[b * N + n] = 0.f;
                            continue;
                        }
                        const Taps tp = taps_at(pr.u, pr.v, h, w);
                        const float* img = prm.conv2 + b * h * w * C3;
                        float* dimg = prm.dconv2 + b * h * w * C3;
                        PointMQ mq = point_mq<false>(img, c1, tp, h, w, C, lane);              // pass 1: M = G^T G, q = G^T d
                        float a0[6], a1[6], jd0, jd1;
                        camera_jacobian(fx, fy, pr.x, pr.y, pr.iZ, a0, a1);
                        depth_jacobian(fx, fy, pr.rx, pr.ry, pr.rz, pr.x, pr.y, pr.iZ, jd0, jd1);
                        // O(K) contractions with this frame's S_cd, S_dc, ghat_d
                        float alpha[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, beta[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, eta = 0.f;
#pragma unroll
                        for (int i = 0; i < KL; ++i) {
                            const int k = lane + 32 * i;
                            if (k < K) {
                                eta = fmaf(sg[6 + k], bl[i], eta);
#pragma unroll
                                for (int m = 0; m < 6; ++m) { alpha[m] = fmaf(Scd[m * K + k], bl[i], alpha[m]); beta[m] = fmaf(Sdc[k * 6 + m], bl[i], beta[m]); }
                            }
                        }
                        eta = warp_sum(eta);
#pragma unroll
                        for (int m = 0; m < 6; ++m) { alpha[m] = warp_sum(alpha[m]); beta[m] = warp_sum(beta[m]); }
                        // 2 x (6+1) algebra (every lane, redundantly).  Point weight of (frame f, point n), as in lm_build_bwd_kernel: Q holds
                        // gamma = b^T S_dd b from frame 0's depth block, so dw is the adjoint of the window-reduced forward (this point's depth
                        // contribution lands in frame 0's block).
                        PointAdjoint ad(a0, a1, jd0, jd1, Scc, sg, alpha, beta, eta, gamma);
                        const float dw = ad.weigh(prm.weight ? __ldg(prm.weight + b * N + n) : 1.f, mq);
                        if (prm.dweight && lane == 0) prm.dweight[b * N + n] = dw;
                        float dJ0[6], dJ1[6], dj0, dj1, vN[8];                 // depth terms of db: vN (6), then tN, sN
                        jacobian_adjoint(mq, ad, sg, eta, dJ0, dJ1, dj0, dj1);
                        depth_terms(a0, a1, jd0, jd1, mq, vN);
                        const float tN = vN[6], sN = vN[7];
                        // pass 2: dd, dG per channel -> dconv1 (summed over the frames), dconv2 (atomics), the coordinate gradient
                        float du, dv;
                        channel_adjoint<false>(img, dimg, c1, sRh, tp, h, w, C, lane, ad, 0.f, [&](int c, float dd) { myDc1[c] += dd; }, du, dv);
                        const GeomGrad gg(pr, fx, fy, Dt, du, dv, dJ0, dJ1, dj0, dj1);
                        if (lane == 0) {
                            sRT[0] += gg.grx * p0; sRT[1] += gg.grx * p1; sRT[2] += gg.grx * p2;
                            sRT[3] += gg.gry * p0; sRT[4] += gg.gry * p1; sRT[5] += gg.gry * p2;
                            sRT[6] += gg.grz * p0; sRT[7] += gg.grz * p1; sRT[8] += gg.grz * p2;
                            sRT[9] += gg.gX; sRT[10] += gg.gY; sRT[11] += gg.gZ;
                        }
                        dDacc += gg.gDt;
#pragma unroll
                        for (int i = 0; i < KL; ++i) {
                            const int k = lane + 32 * i;
                            if (k < K) {
                                float d1 = sN * e[i] + tN * sg[6 + k] + gg.gDt * sW[k];
#pragma unroll
                                for (int m = 0; m < 6; ++m) d1 = fmaf(vN[m], Scd[m * K + k], d1);
                                db[i] += d1;
                                accW[i] = fmaf(gg.gDt, bl[i], accW[i]);
                            }
                        }
                    }
                    // ---- store the frame sums once per point (per frame chunk) ------------------------------------------------------
                    __syncwarp();
                    for (int c = lane; c < C; c += 32) dc1[c] = myDc1[c];
#pragma unroll
                    for (int i = 0; i < KL; ++i) { const int k = lane + 32 * i; if (k < K) prm.dB[gi * K + k] = db[i]; }
                    if (lane == 0) prm.dD[gi] = dDacc;
                    __syncwarp();
                }
            }
            __syncthreads();                                          // commit this chunk's per-frame dR, dT: the warps' sums in a fixed order
            for (int i = tid; i < nfl * 12; i += KB_THREADS) {
                const int fl = i / 12, q = i - fl * 12;
                const float* sRT = sFr + fl * FS + 13 * K + 58 + C;
                float s = 0.f;
                for (int wq = 0; wq < KB_WARPS; ++wq) s += sRT[wq * 12 + q];
                const size_t b = (size_t)wi * nf + fc0 + fl;
                if (q < 9) atomicAdd(prm.dR + b * 9 + q, s); else atomicAdd(prm.dT + b * 3 + q - 9, s);
            }
        }
#pragma unroll
        for (int i = 0; i < KL; ++i) { const int k = lane + 32 * i; if (k < K) atomicAdd(prm.dW + (size_t)wi * K + k, accW[i]); }
        ts = te;
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------------------------
int keyframe_plan(const banet_keyframe_level_t* lv, int num_sms, KeyframePlan* plan)
{
    const int KP = padded_K(lv->K);
    BANET_REQUIRE(lv->K >= 1 && KP > 0, BANET_ERR_UNSUPPORTED, "keyframe build (fp32 SIMT): K=%d > 256 not supported", lv->K);
    BANET_REQUIRE(lv->C <= 2048, BANET_ERR_UNSUPPORTED, "keyframe build: C=%d > 2048", lv->C);
    plan->KP = KP;
    plan->tiles_per_win = (lv->N + KT_PX - 1) / KT_PX;
    plan->total_tiles = (long long)lv->nw * plan->tiles_per_win;
    long long grid = (long long)num_sms * ((KP >= 128) ? 1 : 2);
    if (grid > plan->total_tiles) grid = plan->total_tiles;
    if (grid < 1) grid = 1;
    plan->grid = (int)grid;
    const long long tiles_per_cta = (plan->total_tiles + grid - 1) / grid;
    plan->max_span = (int)((tiles_per_cta + plan->tiles_per_win - 2) / plan->tiles_per_win) + 1;
    plan->slot_floats = KeySlot{lv->K, lv->C}.floats(lv->nf);
    plan->ws_bytes = align_up((size_t)plan->grid * plan->max_span * plan->slot_floats * sizeof(float), 256);
    return BANET_OK;
}

static KeyParams key_params(const banet_keyframe_level_t* lv, const KeyframePlan& plan, const float* R, const float* T, const float* W, void* ws)
{
    KeyParams prm;
    prm.nw = lv->nw; prm.nf = lv->nf; prm.N = lv->N; prm.C = lv->C; prm.K = lv->K; prm.h = lv->h; prm.w = lv->w; prm.c2 = lv->conv2_channels;
    prm.conv1 = lv->conv1; prm.p = lv->p; prm.D = lv->D; prm.B = lv->B; prm.conv2 = lv->conv2; prm.intr = lv->intr;
    prm.R = R; prm.T = T; prm.W = W; prm.weight = lv->weight;
    prm.partials = reinterpret_cast<float*>(ws);
    prm.slot_floats = plan.slot_floats; prm.max_span = plan.max_span; prm.tiles_per_win = plan.tiles_per_win; prm.total_tiles = plan.total_tiles;
    prm.kq_i = 0; prm.kq_j = 0;
    return prm;
}

int keyframe_build(const banet_keyframe_level_t* lv, const KeyframePlan& plan, const float* R, const float* T, const float* W,
                   float* H, float* g, float* rbar_sum, float* nvalid, void* ws, cudaStream_t st)
{
    KeyParams prm = key_params(lv, plan, R, T, W, ws);
    const bool vec4 = (lv->C % 4 == 0) && (lv->conv2_channels % 4 == 0) &&
                      ((reinterpret_cast<uintptr_t>(lv->conv1) | reinterpret_cast<uintptr_t>(lv->conv2)) % 16 == 0);
    int rc;
#define BANET_KEY_DISPATCH(KPV) rc = vec4 ? launch_key_build<KPV, 4>(prm, plan.grid, st) : launch_key_build<KPV, 1>(prm, plan.grid, st)
    switch (plan.KP) {
        case 16:  BANET_KEY_DISPATCH(16); break;
        case 32:  BANET_KEY_DISPATCH(32); break;
        case 64:  BANET_KEY_DISPATCH(64); break;
        case 128: BANET_KEY_DISPATCH(128); break;
        case 256:                                                     // lower-triangle 128-blocks (0,0), (1,0), (1,1)
            rc = BANET_OK;
            for (int blk = 0; blk < 3 && rc == BANET_OK; ++blk) {
                prm.kq_i = blk == 0 ? 0 : 1; prm.kq_j = blk == 2 ? 1 : 0;
                BANET_KEY_DISPATCH(256);
            }
            prm.kq_i = 0; prm.kq_j = 0;
            break;
        default: set_error("keyframe build: bad KP %d", plan.KP); return BANET_ERR_UNSUPPORTED;
    }
#undef BANET_KEY_DISPATCH
    if (rc != BANET_OK) return rc;
    const long long nel = (long long)lv->K * lv->K + (long long)lv->nf * (7 * lv->K + 28 + lv->C);
    int chunks = (int)((nel + 2047) / 2048); if (chunks < 1) chunks = 1; if (chunks > 32) chunks = 32;
    keyframe_reduce_kernel<<<dim3(chunks, grid_y(lv->nw)), 256, 0, st>>>(prm, plan.grid, H, g, rbar_sum, nvalid);
    BANET_CUDA_LAUNCH_CHECK("keyframe_reduce_kernel launch");
    return BANET_OK;
}

static int key_bwd_nfc(int nf, int K, int C)
{
    const size_t budget = 220 * 1024 / sizeof(float), fixed = key_bwd_fixed_floats(K, C), per = key_bwd_frame_floats(K, C);
    if (fixed + per > budget) return 0;
    const size_t n = (budget - fixed) / per;
    return (int)(n < (size_t)nf ? n : (size_t)nf);
}

bool keyframe_build_bwd_supported(int nf, int K, int C) { return K >= 1 && K <= 256 && key_bwd_nfc(nf, K, C) > 0; }

int keyframe_build_bwd(const banet_keyframe_level_t* lv, const float* R, const float* T, const float* W, const float* dH, const float* dg,
                       const float* drbar, int exact_sym, float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW,
                       float* dweight, cudaStream_t st)
{
    const int K = lv->K, C = lv->C, nf = lv->nf;
    const int nfc = key_bwd_nfc(nf, K, C);
    BANET_REQUIRE(nfc > 0, BANET_ERR_UNSUPPORTED, "keyframe build backward: K=%d, C=%d do not fit shared memory", K, C);
    const size_t smem = (key_bwd_fixed_floats(K, C) + (size_t)nfc * key_bwd_frame_floats(K, C)) * sizeof(float);
    void (*kern)(const KeyBwdParams) = K <= 32 ? keyframe_build_bwd_kernel<1> : (K <= 128 ? keyframe_build_bwd_kernel<4> : keyframe_build_bwd_kernel<8>);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("keyframe build backward smem attr: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    KeyBwdParams prm;
    prm.nw = lv->nw; prm.nf = nf; prm.N = lv->N; prm.C = C; prm.K = K; prm.h = lv->h; prm.w = lv->w;
    prm.conv1 = lv->conv1; prm.p = lv->p; prm.D = lv->D; prm.B = lv->B; prm.conv2 = lv->conv2; prm.intr = lv->intr; prm.R = R; prm.T = T; prm.W = W;
    prm.dH = dH; prm.dg = dg; prm.drbar = drbar;
    prm.dconv1 = dconv1; prm.dconv2 = dconv2; prm.dD = dD; prm.dB = dB; prm.dR = dR; prm.dT = dT; prm.dW = dW;
    prm.weight = lv->weight; prm.dweight = dweight;
    prm.exact_sym = exact_sym; prm.nfc = nfc;
    prm.tiles_per_win = (lv->N + KB_TILE - 1) / KB_TILE;
    prm.total_tiles = (long long)lv->nw * prm.tiles_per_win;
    const size_t nb = (size_t)lv->nw * nf;
    cudaMemsetAsync(dconv2, 0, nb * lv->h * lv->w * 3 * C * sizeof(float), st);
    cudaMemsetAsync(dR, 0, nb * 9 * sizeof(float), st);
    cudaMemsetAsync(dT, 0, nb * 3 * sizeof(float), st);
    cudaMemsetAsync(dW, 0, (size_t)lv->nw * K * sizeof(float), st);
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, KB_THREADS, smem) != cudaSuccess || per_sm < 1) { cudaGetLastError(); per_sm = 1; }
    long long grid = (long long)num_sms() * per_sm;
    if (grid > prm.total_tiles) grid = prm.total_tiles;
    kern<<<(int)grid, KB_THREADS, smem, st>>>(prm);
    BANET_CUDA_LAUNCH_CHECK("keyframe_build_bwd_kernel launch");
    return BANET_OK;
}

}  // namespace banet
