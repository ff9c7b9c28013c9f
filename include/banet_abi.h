/*
 * banet_abi.h — C-ABI of libbanet.so: the H100 (sm_90a) drop-in for the BA layer's inner
 * Levenberg–Marquardt loop of frobelbest/BANet.  Plain pointers and sizes only; no torch / TF types.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer (fp32 unless stated), row-major contiguous, laid out exactly
 *     like the reference tensors named beside it; `stream` is a cudaStream_t passed as void*;
 *   - the library allocates nothing and hoards no scratch (contrast reference utils.cu:210-216,
 *     259-296: process-static persistent scratch); the caller owns outputs and workspaces.  The only
 *     process-wide state is the explicit diagnostic tuning struct below (banet_set_tuning; defaults
 *     are the production path) and the thread-local error string; there are no environment knobs;
 *   - every call is asynchronous on `stream` and returns 0 (BANET_OK) or a negative error code;
 *     banet_last_error() gives a thread-local message (reference ignores BLAS status, utils.cu:331);
 *   - per-pair numeric trouble (non-positive pivot, NaN) is reported in a device-side `status[nb]`.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the reference repo).
 */
#ifndef BANET_ABI_H_
#define BANET_ABI_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BANET_ABI_VERSION 1

#define BANET_OK               0
#define BANET_ERR_BAD_ARG     (-1)
#define BANET_ERR_WORKSPACE   (-2)
#define BANET_ERR_CUDA        (-3)
#define BANET_ERR_UNSUPPORTED (-4)

typedef void* banet_stream_t;            /* cudaStream_t */

int         banet_abi_version(void);
const char* banet_last_error(void);
/* 0 if the current CUDA device can run this library (compute capability 9.0), else an error. */
int         banet_device_check(void);
int         banet_num_sms(void);

/* Diagnostic / test knobs (process-wide; defaults = production).  Results never depend on them beyond
 * fp32 summation order. */
typedef struct banet_tuning {
    int tc_generation;      /* 0: default (generation 6 everywhere; lm_build_tc_host.cu has the measurement); 6 / 7: force one wherever it applies (7: F2-only layout + dense grid, TF32X1 / X2) */
    int tc7_force_direct;   /* 1: generation 7 takes its per-tile global-tap fallback for every tile (tests the fallback) */
    int tc7_band_rows;      /* generation 7 walks the 8x8 tiles of a pair in bands of this many tile rows (L2 reuse of the window halos); default 4 */
    int tc6_band_rows;      /* generation 6, dense grid: same walk (tap rows shared by vertically adjacent tiles are re-read from L2, not HBM); 0 = default, 1 = row-major */
    int tc6_l2_hints;       /* generation 6: 0 = default; 1 = no L2 policy; 2 = read-once streams (basis TMA, conv1) evict-first; 3 = 2 + taps evict-last */
    int tc6_tap_prefetch;   /* generation 6: 0 = default; 1 = off; 2 = geometry warps prefetch the tap footprint into L2 ahead of the gather; 3 = 2 with the lower tap row from every pixel */
} banet_tuning_t;
int banet_set_tuning(const banet_tuning_t* t);   /* NULL restores the defaults */
int banet_get_tuning(banet_tuning_t* t);

/* ------------------------------------------------------------------------------------------------
 * (1) Op level — the reference's own native boundary.
 *     Replaces TF op `EquationConstruction` (utils.cu:150-171 op, :219-417 kernel; loaded
 *     bundlenet.py:76-77):   left[b] = sum_n J^T G^T G J,  right[b] = sum_n J^T G^T d.
 *       J [nb,N,2,P]  G [nb,N,C,2]  d [nb,N,C,1]  ->  AtA [nb,P,P]  Atb [nb,P,1]
 * ---------------------------------------------------------------------------------------------- */
size_t banet_eqc_workspace_bytes(int nb, int N, int C, int P);
int    banet_eqc_fwd(const float* J, const float* G, const float* d, int nb, int N, int C, int P,
                     float* AtA, float* Atb, void* ws, size_t ws_bytes, banet_stream_t stream);

/*     Replaces TF op `EquationConstructionGrad` (utils.cu:420-428 op, :465-694 kernel; registered as
 *     the gradient in bundlenet.py:79-82).  With A = G J:
 *       dA = 2 A Ghat + d ghat^T (utils.cu:648-668)   dd = A ghat (:636-645)
 *       dJ = G^T dA (:670-679)                         dG = dA J^T (:681-690)
 *     exact_sym = 0 reproduces the reference (2*A*Ghat); exact_sym = 1 uses A (Ghat + Ghat^T), the
 *     true adjoint for a non-symmetric upstream gradient.  No workspace needed. */
int    banet_eqc_bwd(const float* J, const float* G, const float* d,
                     const float* gAtA, const float* gAtb, int nb, int N, int C, int P, int exact_sym,
                     float* dJ, float* dG, float* dd, banet_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * (2) Pre-steps of a level.
 * ---------------------------------------------------------------------------------------------- */
/* BundleNet.computeCoordinates (bundlenet.py:112-120; un-normalised legacy/ba.py:27-34).
 *   points [nb,N,2], intr [nb,4]=(fx,fy,ox,oy) -> p [nb,3,N]   (L2-normalised iff normalize!=0) */
int banet_compute_coordinates(const float* points, const float* intr, int nb, int N, int normalize,
                              float* p, banet_stream_t stream);
/* BundleNet.grad_fixed + concat (bundlenet.py:92-100, 388-389), optionally fused with the
 * half-swap pairing of :386 (swap_halves!=0: output pair b reads input pair (b + nb/2) % nb).
 *   F [nb,h,w,C] -> conv2 [nb,h,w,3C] = [F | gradx | grady] */
int banet_grad_fixed_concat(const float* F, int nb, int h, int w, int C, int swap_halves,
                            float* conv2, banet_stream_t stream);
/* tf.contrib.resampler.resampler (call sites bundlenet.py:290,320,343,344,385): bilinear, zero outside.
 *   data [nb,h,w,C], xy [nb,N,2] (sampled at xy*coord_scale) -> out [nb,N,C] */
int banet_resample(const float* data, const float* xy, float coord_scale, int nb, int h, int w, int C, int N,
                   float* out, banet_stream_t stream);

/* The legacy sampler (legacy/utils_python.py:61-117 `interpolate2d`, :177-232 `interpolate2d2`): bilinear with CLAMPED tap indices;
 * mask [nb,N] (optional, may be NULL) = the in-bounds test of :114-116.  Same layouts as banet_resample. */
int banet_interpolate2d(const float* data, const float* xy, float coord_scale, int nb, int h, int w, int C, int N,
                        float* out, float* mask, banet_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * (3) Layer level — one LM iteration = BundleNet.BundleIteration (bundlenet.py:193-278) or
 *     BundleNet.CameraIteration (:122-191) when K == 0 / B == NULL.
 * ---------------------------------------------------------------------------------------------- */
typedef struct banet_level {
    int nb, N, C, K;          /* pairs, points per pair, feature channels, depth bases (0 = pose only) */
    int h, w;                 /* conv2 map size at this level */
    int conv2_channels;       /* 3*C: [F2|gx|gy] as in the reference; C: F2 only, gradients derived on the fly */
    const float* conv1;       /* [nb,N,C]      bundlenet.py:385 */
    const float* conv2;       /* [nb,h,w,conv2_channels]  :386-389 */
    const float* intr;        /* [nb,4] fx,fy,ox,oy at this level (reference tiles them to [nb,N], :379-382) */
    const float* p;           /* [nb,3,N]      :358 */
    const float* D;           /* [nb,N,1]      :343 */
    const float* B;           /* [nb,N,K] or NULL  :344 */
    int grid_w, grid_h;       /* locality hint, results do not depend on it: 0,0 = unstructured point list; otherwise the N points
                                 are the row-major raster grid x<grid_w, y<grid_h (N == grid_w*grid_h) and the kernels walk it in
                                 8x8 tiles so that every conv2 texel is fetched from HBM about once */
} banet_level_t;

#define BANET_PREC_AUTO    (-1)   /* the level-wise policy (TF32_LEVELWISE) where the tensor-core path applies (K in {32,64,128}, C in {64,128}), else FP32_SIMT */
#define BANET_PREC_FP32_SIMT 0   /* every contraction in fp32 FFMA (reference-exact arithmetic type)   */
#define BANET_PREC_TF32X1    1   /* B^T diag(s) B on tcgen05 kind::tf32: basis truncated by the tensor core, s*b rounded to nearest */
#define BANET_PREC_TF32X2    2   /* split-A two-pass tf32: b = trunc(b) + (b - trunc(b)); only s*b's rounding remains             */
#define BANET_PREC_TF32X3    3   /* three passes: also s*b = hi + lo; the dropped lo*lo term is ~2^-22: fp32-grade sums          */
#define BANET_PREC_TF32_LEVELWISE 4 /* per level: TF32X3 below 65536 points per pair, TF32X1 above (FP32_SIMT where tensor cores do not apply) */

/* Normal equations + damping statistics of one iteration (bundlenet.py:206-239, 259-263 and the
 * mean-|diff| of :243), fused: J, G, d are never materialised.
 *   R [nb,3,3], T [nb,3,1], W [nb,K,1] ->
 *   H [nb,P,P] (= AtA), g [nb,P] (= Atb), rbar_sum [nb,C] (= sum_n |diff|, NOT yet divided by N),
 *   nvalid [nb] (in-bounds point count, as float).   P = 6 + K. */
size_t banet_lm_build_workspace_bytes(const banet_level_t* lv, int precision);
int    banet_lm_build(const banet_level_t* lv, const float* R, const float* T, const float* W,
                      int precision, float* H, float* g, float* rbar_sum, float* nvalid,
                      void* ws, size_t ws_bytes, banet_stream_t stream);

/* lambda prediction (bundlenet.py:241-253; pose-only :165-173): rbar = rbar_sum/N, 5 dense layers
 * C->2C->4C->2C->C->1 (selu x4, tanh), lambda = base * ||rbar||_2^(2+h).
 *   mlp_weights: the 5 filters [cin,cout] then... see banet_mlp_param_count(); packed
 *   [W1,b1,W2,b2,...,W5,b5] in one buffer, W_i row-major [cin,cout] (TF conv1d filter [1,cin,cout]).
 *   base: l2_regularizer_base (1000 in :393; pass 1 for CameraIteration, which ignores it). */
size_t banet_mlp_param_count(int C);
int    banet_lm_lambda(const float* rbar_sum, int nb, int N, int C, const float* mlp_weights, float base,
                       float* lambda_out, banet_stream_t stream);

typedef struct banet_solve_opts {
    float damping_eps;          /* 1e-5  (bundlenet.py:182,266) */
    int   undamped_last;        /* 1 for BundleIteration (:266 leaves the last depth coefficient undamped); 0 for CameraIteration */
    int   vmatrix_batch_scramble; /* 0: per-pair V; 1: reproduce the axis-0 stack of bundlenet.py:45 literally (nb>1 interleaves pairs) */
} banet_solve_opts_t;

/* Damping + solve + update (bundlenet.py:264-276; pose-only :181-190).  tf.matrix_solve (LU) is
 * replaced by an in-shared-memory Cholesky (the damped normal matrix is SPD).
 *   H,g,lambda[nb], R,T,W -> R',T',W' (may alias the inputs), delta [nb,P] (the solution, optional/NULL),
 *   status [nb] int32: 0 ok, 1 non-positive pivot (matrix not SPD), 2 non-finite input. */
size_t banet_lm_solve_workspace_bytes(int nb, int K);
int    banet_lm_solve_update(const float* H, const float* g, const float* lambda, int nb, int K,
                             const banet_solve_opts_t* opts,
                             const float* R, const float* T, const float* W,
                             float* R_out, float* T_out, float* W_out, float* delta, int32_t* status,
                             void* ws, size_t ws_bytes, banet_stream_t stream);

/* banet_lm_lambda + banet_lm_solve_update in ONE launch (blocked Cholesky with the right-hand side as an extra row): what banet_lm_run
 * executes per iteration.  mlp_weights NULL: lambda_in [nb] is used instead of the MLP.  lambda_out [nb] always receives the damping used.
 * R_out/T_out/W_out may alias R/T/W.  opts->vmatrix_batch_scramble must be 0 (that option needs every pair's solution first). */
int    banet_lm_step(const float* H, const float* g, const float* rbar_sum, int nb, int N, int C, int K,
                     const float* mlp_weights, float base, const float* lambda_in, const banet_solve_opts_t* opts,
                     const float* R, const float* T, const float* W, float* R_out, float* T_out, float* W_out,
                     float* delta, float* lambda_out, int32_t* status, banet_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * (3b) Backward of one LM iteration — the gradient signature of the reference's BA layer: TF autodiff of
 *      bundlenet.py:193-278 with the registered op gradient EquationConstructionGrad (bundlenet.py:79-82,
 *      utils.cu:465-694), w.r.t. every float input it differentiates: conv1, conv2, D, B, R, T, W (and, through
 *      lambda, the MLP variables).  J, G, d and the tiled upstream gradients of utils.cu:613-617 are never formed.
 * ---------------------------------------------------------------------------------------------- */
/* Backward of banet_lm_build.  dH [nb,P,P] (as the solve's backward emits it: not symmetric), dg [nb,P],
 * drbar_sum [nb,C]  ->  dconv1 [nb,N,C], dconv2 [nb,h,w,3C], dD [nb,N,1], dB [nb,N,K], dR [nb,3,3], dT [nb,3,1],
 * dW [nb,K,1]; every output is overwritten.  conv2 must be the reference's [F2|gx|gy] layout (the F2-only layout
 * adds banet_grad_fixed_concat_bwd).  exact_sym as in banet_eqc_bwd (0 = the reference's 2*A*Ghat). */
int    banet_lm_build_bwd(const banet_level_t* lv, const float* R, const float* T, const float* W,
                          const float* dH, const float* dg, const float* drbar_sum, int exact_sym,
                          float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW,
                          banet_stream_t stream);
/* Backward of banet_lm_solve_update: gradients of (R',T',W') [dR_out,dT_out,dW_out] -> dH [nb,P,P], dg [nb,P],
 * dlambda [nb], dR, dT, dW.  `delta` [nb,P] is the solution the forward call returned.  Pairs whose forward step was
 * skipped (status != 0, delta = 0) pass the pose/depth gradients through and get zero dH, dg, dlambda.
 * opts->vmatrix_batch_scramble must be 0. */
int    banet_lm_solve_update_bwd(const float* H, const float* g, const float* lambda, const float* delta, int nb, int K,
                                 const banet_solve_opts_t* opts, const float* R, const float* T,
                                 const float* dR_out, const float* dT_out, const float* dW_out,
                                 float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW,
                                 banet_stream_t stream);
/* Backward of banet_grad_fixed_concat (transposed REFLECT stencil + the half swap): dconv2 [nb,h,w,3C] -> dF [nb,h,w,C]. */
int    banet_grad_fixed_concat_bwd(const float* dconv2, int nb, int h, int w, int C, int swap_halves,
                                   float* dF, banet_stream_t stream);

/* Backward of banet_resample w.r.t. the sampled map (the coordinates are constants on this path, bundlenet.py:343-344, 385):
 *   dout [nb,N,C] -> ddata [nb,h,w,C] (overwritten). */
int    banet_resample_bwd(const float* dout, const float* xy, float coord_scale, int nb, int h, int w, int C, int N,
                          float* ddata, banet_stream_t stream);
/* Backward of banet_depth_compose: dout [nb,M] -> dbasis [nb,M,K], dW [nb,K,1] (overwritten); d init_depth = dout. */
int    banet_depth_compose_bwd(const float* dout, const float* basis, const float* W, int nb, int M, int K,
                               float* dbasis, float* dW, banet_stream_t stream);

/* Whole coarse-to-fine solve: for each level, `iters_per_level` iterations of
 * build -> lambda -> solve/update, with W carried across levels (the level loop of
 * bundlenet.py:376-399 with the iteration count of legacy/ba.py:106-121).
 *   mlp_weights[l]: packed lambda-MLP of level l, or NULL with lambda_fixed >= 0 to bypass the MLP.
 *   R,T,W are updated in place.  status [nb] accumulates (bitwise or) the per-iteration status. */
size_t banet_lm_run_workspace_bytes(const banet_level_t* levels, int nlevels, int precision);
int    banet_lm_run(const banet_level_t* levels, int nlevels, int iters_per_level,
                    const float* const* mlp_weights, float l2_regularizer_base, float lambda_fixed,
                    const banet_solve_opts_t* opts, int precision,
                    float* R, float* T, float* W, int32_t* status,
                    void* ws, size_t ws_bytes, banet_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * (3c) Joint keyframe window — an EXTENSION (SURVEY.md section 8f-4), not in the reference: its BA layer is 2-view (one pose and one W
 *      per pair, bundlenet.py:193-278) and BA-Net's 5-frame case runs as 4 independent pairs (legacy/seq_example.py).  Here the nb = nf
 *      pairs of every level are (keyframe -> frame f) and share the keyframe's depth D + B.W: 6 nf + K unknowns, block-arrow normal
 *      matrix (per-pair pose blocks and pose-depth couplings from banet_lm_build, depth block and depth right-hand side summed over the
 *      frames), lambda from the mean |residual| over all points of all frames through the same MLP (bundlenet.py:241-253), the
 *      reference's damping (:264-266, last depth coefficient undamped), ONE solve, per-frame SE(3) update (:269-275), shared W update.
 *      Same arguments as banet_lm_run.  conv1, p, D, B of a level hold the keyframe's tensors once per frame (the [nb,...] layout).
 *      W [nf,K,1]: frame 0's row is the window's W on entry (it is broadcast), every row holds the shared result on exit.
 *      status [nf]: the window's status (a skipped step skips every frame).  6 nf + K must fit the fused dense solve: it factors in fp64 up to
 *      218 unknowns and in fp32 up to 325 (at C = 128; 220 and 329 with lambda_fixed), and rejects larger windows with BANET_ERR_UNSUPPORTED
 *      (nf <= 15 in fp64 and nf <= 32 at all at K = 128).  Section (3d) has no such limit. */
size_t banet_lm_window_run_workspace_bytes(const banet_level_t* levels, int nlevels, int precision);
int    banet_lm_window_run(const banet_level_t* levels, int nlevels, int iters_per_level,
                           const float* const* mlp_weights, float l2_regularizer_base, float lambda_fixed,
                           const banet_solve_opts_t* opts, int precision,
                           float* R, float* T, float* W, int32_t* status,
                           void* ws, size_t ws_bytes, banet_stream_t stream);

/* One window iteration after the build, with the damping given (the training path of the window; SURVEY.md section 8f-4, DESIGN.md §7 item 6):
 * the step banet_lm_window_run takes per iteration with lambda_fixed -- assembly of the block-arrow system, damping (:264-266), one solve,
 * per-frame SE(3) update (:269-275), shared W update (:276) -- and the same bits for the same lambda.
 *   H [nf,P,P], g [nf,P]: banet_lm_build with nb = nf (P = 6 + K); lambda [1]; R [nf,3,3], T [nf,3,1], W [K,1] (shared)
 *   -> R_out, T_out, W_out [K,1] (may alias the inputs), delta [6 nf + K] (the joint solution: frame f's pose step at 6f, the depth step at
 *   6 nf; the backward needs it), status [nf] (the window's status for every frame; a skipped step skips every frame: delta = 0).
 * 6 nf + K must fit the fused dense solve: fp64 up to 220 unknowns, fp32 up to 329, BANET_ERR_UNSUPPORTED beyond. */
size_t banet_lm_window_solve_update_workspace_bytes(int nf, int K);
int    banet_lm_window_solve_update(const float* H, const float* g, const float* lambda, int nf, int K, const banet_solve_opts_t* opts,
                                    const float* R, const float* T, const float* W, float* R_out, float* T_out, float* W_out,
                                    float* delta, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream);
/* Its backward: gradients of (R',T',W') [dR_out [nf,3,3], dT_out [nf,3,1], dW_out [K,1]] -> dH [nf,P,P] (not symmetric, as
 * banet_lm_build_bwd takes it), dg [nf,P], dlambda [1], dR, dT, dW [K,1]; every output is overwritten.  dW = dW_out: the build's share of
 * dW comes from banet_lm_build_bwd.  A skipped step (status != 0, delta = 0) gets zero dH, dg, dlambda and passes dR_out, dT_out, dW_out
 * through, as banet_lm_solve_update_bwd does.  The backward factors the damped system in fp64 up to 6 nf + K = 222 and in fp32 up to 332;
 * the forward's fused solve switches to fp32 above 220 unknowns and rejects more than 329. */
size_t banet_lm_window_solve_update_bwd_workspace_bytes(int nf, int K);
int    banet_lm_window_solve_update_bwd(const float* H, const float* g, const float* lambda, const float* delta, int nf, int K,
                                        const banet_solve_opts_t* opts, const float* R, const float* T,
                                        const float* dR_out, const float* dT_out, const float* dW_out,
                                        float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW,
                                        void* ws, size_t ws_bytes, banet_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * (3d) Batches of keyframe windows — the same extension as (3c), nw windows per call, each solved through its block-arrow structure:
 *      the per-frame 6x6 pose blocks are eliminated (Schur complement) and only the K x K depth system is factored, so nf is limited by
 *      the workspace only.  The maths is (3c)'s: lambda from the window's mean |residual| over its nf N points through the MLP
 *      (bundlenet.py:241-253), damping of every diagonal entry but the last depth coefficient (:264-266), per-frame SE(3) update (:269-275),
 *      shared W update (:276); results agree with (3c) to fp32 rounding, not bit for bit (a different factorisation).
 *      Conventions: pair w*nf + f is (keyframe of window w -> frame f); H, g, R, T, conv1 ... of a level are per pair ([nw*nf,...]: the
 *      keyframe's tensors once per frame), W [nw,K,1] and lambda [nw] per window, status [nw*nf] (a window's status for each of its frames:
 *      0 ok, 1 non-positive pivot in a frame's 6x6 block or in the depth system, 2 non-finite input; a skipped window has delta = 0 and
 *      keeps its R, T, W; other windows are not affected).  delta [nw, 6 nf + K]: frame f's pose step at 6f, the depth step at 6 nf.
 *      The depth system is factored in fp64 while it fits shared memory (K <= 211 at C = 128, K <= 215 with lambda given), else in fp32;
 *      K <= 256 (the build's range).  Every sum is taken in a fixed order: bit-reproducible, independent of the workspace's contents.
 *      Argument errors (null pointers, nw, nf, K <= 0, vmatrix_batch_scramble != 0, nb != nw*nf: BANET_ERR_BAD_ARG; K out of range:
 *      BANET_ERR_UNSUPPORTED; workspace too small: BANET_ERR_WORKSPACE) are reported before any CUDA call.
 * ---------------------------------------------------------------------------------------------- */
/* Whole coarse-to-fine solve of nw windows: banet_lm_window_run's arguments plus nw; levels[l].nb == nw*nf.  Each iteration is one build
 * launch (all nw*nf pairs) and one step launch (all nw windows).  R [nw*nf,3,3], T [nw*nf,3,1], W [nw,K,1] are updated in place; status
 * [nw*nf] accumulates (bitwise or).  The per-pair copies of W the build reads live in the workspace. */
size_t banet_lm_window_batch_run_workspace_bytes(const banet_level_t* levels, int nlevels, int nw, int precision);
int    banet_lm_window_batch_run(const banet_level_t* levels, int nlevels, int nw, int iters_per_level,
                                 const float* const* mlp_weights, float l2_regularizer_base, float lambda_fixed,
                                 const banet_solve_opts_t* opts, int precision,
                                 float* R, float* T, float* W, int32_t* status,
                                 void* ws, size_t ws_bytes, banet_stream_t stream);

/* One iteration of nw windows after the build, with the damping given (the training path; banet_lm_window_solve_update per window):
 *   H [nw*nf,P,P], g [nw*nf,P] (banet_lm_build with nb = nw*nf, P = 6 + K), lambda [nw], R [nw*nf,3,3], T [nw*nf,3,1], W [nw,K,1]
 *   -> R_out, T_out, W_out (may alias the inputs), delta [nw, 6 nf + K] (the backward needs it), status [nw*nf]. */
size_t banet_lm_window_batch_solve_update_workspace_bytes(int nw, int nf, int K);
int    banet_lm_window_batch_solve_update(const float* H, const float* g, const float* lambda, int nw, int nf, int K, const banet_solve_opts_t* opts,
                                          const float* R, const float* T, const float* W, float* R_out, float* T_out, float* W_out,
                                          float* delta, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream);
/* Its backward: gradients of (R',T',W') [dR_out [nw*nf,3,3], dT_out [nw*nf,3,1], dW_out [nw,K,1]] -> dH [nw*nf,P,P] (not symmetric, as
 * banet_lm_build_bwd takes it), dg [nw*nf,P], dlambda [nw], dR, dT, dW [nw,K,1]; every output is overwritten.  Per window these are
 * banet_lm_window_solve_update_bwd's values: the solve backward (the (1 + lambda) factor on the damped diagonal) composed with the
 * assembly's adjoint, the depth block's gradient given to every frame, written per pair.  dW = dW_out.  A skipped window (the forward's
 * status, re-derived from H, g, lambda) gets zero dH, dg, dlambda and passes dR_out, dT_out, dW_out through. */
size_t banet_lm_window_batch_solve_update_bwd_workspace_bytes(int nw, int nf, int K);
int    banet_lm_window_batch_solve_update_bwd(const float* H, const float* g, const float* lambda, const float* delta, int nw, int nf, int K,
                                              const banet_solve_opts_t* opts, const float* R, const float* T,
                                              const float* dR_out, const float* dT_out, const float* dW_out,
                                              float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW,
                                              void* ws, size_t ws_bytes, banet_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * (4) The legacy pose-only keyframe tracker loop: legacy/ba.py:83-145 (`Tracker.trackTF`) with CameraIteration (:147-214) or, with
 *     early termination, CameraIteration2 (:226-345: lambda-MLP step, residual re-evaluated at the updated pose, step kept only if it
 *     decreased) — accept / reject and the per-level termination test run on the device, per pair, without host synchronisation.
 *     levels[l]: pose-only (K = 0, B NULL), conv2 = [F2|gx|gy]; level_iters[l] = maximum iterations at level l.
 *     iters_done [nlevels,nb] (optional): CameraIteration2 calls each pair actually made per level.
 *     valid_ratio [nb]: what the reference returns as `ratio` — N / valid of the last executed CameraIteration2, or valid / N (plain).
 * ---------------------------------------------------------------------------------------------- */
typedef struct banet_legacy_opts {
    int   early_termination;     /* legacy/ba.py:5  (True)                  */
    float angle_change;          /* legacy/ba.py:6  0.002 * (3.14 / 180)    */
    float translation_change;    /* legacy/ba.py:7  0.0002                  */
    float residual_ratio;        /* legacy/ba.py:8  1.0                     */
} banet_legacy_opts_t;
size_t banet_lm_track_legacy_workspace_bytes(const banet_level_t* levels, int nlevels);
int    banet_lm_track_legacy(const banet_level_t* levels, int nlevels, const int* level_iters, const float* const* mlp_weights,
                             const banet_legacy_opts_t* opts, float* R, float* T, int32_t* iters_done, float* valid_ratio,
                             int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream);

/* Final depth composition of BundleResize (bundlenet.py:397): out = init_depth + basis . W
 *   basis [nb,M,K] (M = h/2*w/2), W [nb,K,1], init_depth [nb,M] -> out [nb,M] */
int banet_depth_compose(const float* init_depth, const float* basis, const float* W, int nb, int M, int K,
                        float* out, banet_stream_t stream);

/* Diagnostic (not part of the reference's interface): one 64-pixel k-tile through the TMA + tcgen05 building
 * blocks of the tensor-core build path.  A [64,128], R [64,160] -> D [128,160] = A^T R.
 * mode 0: single tf32 pass; mode 1: split-A two-pass.  use_rna: round R to tf32 (nearest) first.
 * repeat: accumulate the same tile `repeat` times into TMEM (probes the accumulator's rounding). */
int banet_tc_selftest(const float* A, const float* R, float* D, int mode, int use_rna, int repeat, banet_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* BANET_ABI_H_ */
