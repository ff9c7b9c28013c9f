// extern "C" entry points of libbanet.so (see include/banet_abi.h) + run_solve, the coarse-to-fine schedule of the four whole-solve entries.
#include "common.cuh"
#include "lm_build.h"
#include <string.h>
#include <algorithm>
#include <type_traits>

namespace banet {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int num_sms()
{
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return kMaxSMs; }
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { cudaGetLastError(); return kMaxSMs; }
    return n;
}

// the robust loss of a level: a known kind, and a finite positive scale when it is not BANET_ROBUST_NONE
static int check_robust(const banet_level_t* lv, const char* who)
{
    BANET_REQUIRE(lv->robust == BANET_ROBUST_NONE || lv->robust == BANET_ROBUST_HUBER || lv->robust == BANET_ROBUST_CAUCHY, BANET_ERR_BAD_ARG,
                  "%s: robust=%d must be BANET_ROBUST_NONE (0), BANET_ROBUST_HUBER (1) or BANET_ROBUST_CAUCHY (2)", who, lv->robust);
    BANET_REQUIRE(lv->robust == BANET_ROBUST_NONE || (isfinite(lv->robust_scale) && lv->robust_scale > 0.f), BANET_ERR_BAD_ARG,
                  "%s: robust_scale=%g must be finite and > 0 with a robust loss", who, (double)lv->robust_scale);
    return BANET_OK;
}

static int check_level(const banet_level_t* lv, const char* who)
{
    BANET_REQUIRE(lv, BANET_ERR_BAD_ARG, "%s: null level", who);
    BANET_REQUIRE(lv->nb > 0 && lv->N > 0 && lv->C > 0 && lv->K >= 0 && lv->h >= 2 && lv->w >= 2, BANET_ERR_BAD_ARG,
                  "%s: bad shape nb=%d N=%d C=%d K=%d h=%d w=%d", who, lv->nb, lv->N, lv->C, lv->K, lv->h, lv->w);
    BANET_REQUIRE(lv->conv2_channels == 3 * lv->C || lv->conv2_channels == lv->C, BANET_ERR_BAD_ARG,
                  "%s: conv2_channels=%d must be 3*C (reference layout) or C (F2 only)", who, lv->conv2_channels);
    BANET_REQUIRE(lv->conv1 && lv->conv2 && lv->intr && lv->p && lv->D, BANET_ERR_BAD_ARG, "%s: null tensor", who);
    BANET_REQUIRE(lv->feature_dtype == BANET_DTYPE_F32 || lv->feature_dtype == BANET_DTYPE_BF16, BANET_ERR_BAD_ARG,
                  "%s: feature_dtype=%d must be BANET_DTYPE_F32 (0) or BANET_DTYPE_BF16 (1)", who, lv->feature_dtype);
    BANET_REQUIRE(lv->basis_dtype == BANET_DTYPE_F32 || lv->basis_dtype == BANET_DTYPE_BF16, BANET_ERR_BAD_ARG,
                  "%s: basis_dtype=%d must be BANET_DTYPE_F32 (0) or BANET_DTYPE_BF16 (1)", who, lv->basis_dtype);
    BANET_REQUIRE(lv->K == 0 || lv->B, BANET_ERR_BAD_ARG, "%s: K=%d but B is null", who, lv->K);
    BANET_REQUIRE((long long)lv->h * lv->w * lv->conv2_channels < (1LL << 40), BANET_ERR_BAD_ARG, "%s: map too large", who);
    BANET_REQUIRE((lv->grid_w == 0 && lv->grid_h == 0) || (lv->grid_w > 0 && lv->grid_h > 0 && (long long)lv->grid_w * lv->grid_h == lv->N),
                  BANET_ERR_BAD_ARG, "%s: grid %dx%d does not match N=%d", who, lv->grid_w, lv->grid_h, lv->N);
    return check_robust(lv, who);
}

// Level-wise policy (BANET_PREC_TF32_LEVELWISE; measured motivation in DESIGN.md §4): the rounding error of H averages out as
// 1/sqrt(N), so the coarse levels carry nearly all of a solve's error and nearly none of its time: TF32X3 (fp32-grade) below
// 65536 points per pair, single-pass TF32X1 above.
static int levelwise_mode(const banet_level_t* lv) { return lv->N < 65536 ? BANET_PREC_TF32X3 : BANET_PREC_TF32X1; }

int resolve_precision(const banet_level_t* lv, int precision)
{
    if (precision == BANET_PREC_AUTO) {
        // AUTO = the level-wise policy: measured on the cfg2 bench workload (32 pairs, 20 iterations, against the FP32 path; profiles/r02_*):
        // W 4.2e-6 / depth 5.8e-7 where TF32X2 everywhere gives 2.6e-4 / 3.5e-5 and TF32X1 3.6e-4 / 5.0e-5 -- and it is the fastest of the three.
        if (!tc_supported(lv)) return BANET_PREC_FP32_SIMT;
        return lv->K == 128 ? levelwise_mode(lv) : BANET_PREC_TF32X2;       // K = 64 / 32: the single-pass mode is not instantiated
    }
    if (precision == BANET_PREC_TF32_LEVELWISE) {
        if (!tc_supported(lv)) return BANET_PREC_FP32_SIMT;
        return levelwise_mode(lv);
    }
    if (precision == BANET_PREC_FP32_SIMT) return precision;
    if (precision == BANET_PREC_TF32X1 || precision == BANET_PREC_TF32X2 || precision == BANET_PREC_TF32X3) {
        if (!tc_supported(lv)) {
            if (lv->conv2_channels == lv->C && lv->w >= 65536)        // tc_supported(): the F2-only gather packs tap columns in 16 bits
                set_error("precision mode %d (tensor cores) needs w < 65536 in the F2-only layout (tap columns are packed in 16 bits); got w=%d",
                          precision, lv->w);
            else
                set_error("precision mode %d (tensor cores) needs K=128, C in {64,128} and 16-B aligned tensors; got K=%d C=%d", precision, lv->K, lv->C);
            return BANET_ERR_UNSUPPORTED;
        }
        return precision;
    }
    set_error("unknown precision mode %d", precision);
    return BANET_ERR_BAD_ARG;
}

int plan_for(const banet_level_t* lv, int resolved, BuildPlan* plan)
{
    return resolved == BANET_PREC_FP32_SIMT ? build_plan(lv, num_sms(), plan) : build_plan_tc(lv, num_sms(), plan);
}

int build_dispatch(const banet_level_t* lv, int resolved, const BuildPlan& plan, const float* R, const float* T, const float* W,
                   float* H, float* g, float* rbar_sum, float* nvalid, void* ws, cudaStream_t st)
{
    if (resolved == BANET_PREC_FP32_SIMT) return lm_build_simt(lv, plan, R, T, W, H, g, rbar_sum, nvalid, ws, st);
    return lm_build_tc(lv, plan, resolved, R, T, W, H, g, rbar_sum, nvalid, ws, st);
}

}  // namespace banet

using namespace banet;

extern "C" int banet_abi_version(void) { return BANET_ABI_VERSION; }
extern "C" const char* banet_last_error(void) { return g_err; }
extern "C" int banet_num_sms(void) { return num_sms(); }

extern "C" int banet_set_tuning(const banet_tuning_t* t)
{
    const banet_tuning_t def = {0, 0, 0};
    if (!t) { set_tuning(def); return BANET_OK; }
    BANET_REQUIRE(t->tc6_band_rows >= 0 && t->tc6_l2_hints >= 0 && t->tc6_l2_hints <= 3 && t->tc6_tap_prefetch >= 0 && t->tc6_tap_prefetch <= 3, BANET_ERR_BAD_ARG,
                  "set_tuning: tc6_band_rows >= 0, tc6_l2_hints and tc6_tap_prefetch in 0..3");
    set_tuning(*t);
    return BANET_OK;
}
extern "C" int banet_get_tuning(banet_tuning_t* t)
{
    BANET_REQUIRE(t, BANET_ERR_BAD_ARG, "get_tuning: null");
    *t = tuning();
    return BANET_OK;
}

extern "C" int banet_device_check(void)
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) { cudaGetLastError(); set_error("no CUDA device: %s", cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    int major = 0, minor = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
    BANET_REQUIRE(major == 9 && minor == 0, BANET_ERR_UNSUPPORTED, "device compute capability %d.%d; this library is built for sm_90a only", major, minor);
    return BANET_OK;
}

// -------------------------------------------------------------------------------------------------
extern "C" size_t banet_lm_build_workspace_bytes(const banet_level_t* lv, int precision)
{
    if (!lv || check_robust(lv, "lm_build_workspace_bytes")) return 0;
    const int res = resolve_precision(lv, precision);
    if (res < 0) return 0;
    BuildPlan plan;
    if (plan_for(lv, res, &plan) != BANET_OK) return 0;
    return plan.ws_bytes;
}

extern "C" int banet_lm_build(const banet_level_t* lv, const float* R, const float* T, const float* W, int precision,
                              float* H, float* g, float* rbar_sum, float* nvalid, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    int rc = check_level(lv, "lm_build");
    if (rc) return rc;
    BANET_REQUIRE(R && T && H && g && rbar_sum && nvalid, BANET_ERR_BAD_ARG, "lm_build: null pointer");
    BANET_REQUIRE(lv->K == 0 || W, BANET_ERR_BAD_ARG, "lm_build: K=%d but W is null", lv->K);
    const int res = resolve_precision(lv, precision);
    if (res < 0) return res;
    BuildPlan plan;
    rc = plan_for(lv, res, &plan);
    if (rc) return rc;
    BANET_REQUIRE(ws && ws_bytes >= plan.ws_bytes, BANET_ERR_WORKSPACE, "lm_build: workspace %zu < %zu bytes", ws_bytes, plan.ws_bytes);
    return build_dispatch(lv, res, plan, R, T, W, H, g, rbar_sum, nvalid, ws, (cudaStream_t)stream);
}

extern "C" size_t banet_mlp_param_count(int C) { return (size_t)20 * C * C + (size_t)10 * C + 1; }

extern "C" int banet_lm_lambda(const float* rbar_sum, int nb, int N, int C, const float* mlp_weights, float base,
                               float* lambda_out, banet_stream_t stream)
{
    BANET_REQUIRE(rbar_sum && mlp_weights && lambda_out && nb > 0 && N > 0 && C > 0, BANET_ERR_BAD_ARG, "lm_lambda: bad argument");
    return lm_lambda(rbar_sum, nb, N, C, mlp_weights, base, lambda_out, (cudaStream_t)stream);
}

extern "C" size_t banet_lm_solve_workspace_bytes(int nb, int K)
{
    if (nb <= 0 || K < 0) return 0;
    return align_up((size_t)nb * (6 + K) * sizeof(float), 256);
}

extern "C" int banet_lm_solve_update(const float* H, const float* g, const float* lambda, int nb, int K,
                                     const banet_solve_opts_t* opts, const float* R, const float* T, const float* W,
                                     float* R_out, float* T_out, float* W_out, float* delta, int32_t* status,
                                     void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(H && g && lambda && opts && R && T && R_out && T_out && status, BANET_ERR_BAD_ARG, "lm_solve_update: null pointer");
    BANET_REQUIRE(nb > 0 && K >= 0, BANET_ERR_BAD_ARG, "lm_solve_update: bad shape nb=%d K=%d", nb, K);
    BANET_REQUIRE(K == 0 || (W && W_out), BANET_ERR_BAD_ARG, "lm_solve_update: K=%d but W is null", K);
    if (!delta) {
        BANET_REQUIRE(ws && ws_bytes >= banet_lm_solve_workspace_bytes(nb, K), BANET_ERR_WORKSPACE,
                      "lm_solve_update: delta is null and workspace %zu < %zu bytes", ws_bytes, banet_lm_solve_workspace_bytes(nb, K));
        delta = reinterpret_cast<float*>(ws);
    }
    return lm_solve_update(H, g, lambda, nb, K, *opts, R, T, W, R_out, T_out, W_out, delta, status, 0, (cudaStream_t)stream);
}

extern "C" int banet_lm_step(const float* H, const float* g, const float* rbar_sum, int nb, int N, int C, int K, const float* mlp_weights, float base,
                             const float* lambda_in, const banet_solve_opts_t* opts, const float* R, const float* T, const float* W,
                             float* R_out, float* T_out, float* W_out, float* delta, float* lambda_out, int32_t* status, banet_stream_t stream)
{
    BANET_REQUIRE(H && g && opts && R && T && R_out && T_out && delta && lambda_out && status && nb > 0 && K >= 0, BANET_ERR_BAD_ARG, "lm_step: bad argument");
    BANET_REQUIRE((mlp_weights && rbar_sum && N > 0 && C > 0) || lambda_in, BANET_ERR_BAD_ARG, "lm_step: needs lambda-MLP weights + rbar_sum, or lambda_in");
    BANET_REQUIRE(K == 0 || (W && W_out), BANET_ERR_BAD_ARG, "lm_step: K=%d but W is null", K);
    BANET_REQUIRE(!opts->vmatrix_batch_scramble, BANET_ERR_UNSUPPORTED, "lm_step: vmatrix_batch_scramble needs the separate banet_lm_solve_update");
    return lm_step(H, g, rbar_sum, nb, N, C > 0 ? C : 1, K, mlp_weights, base, mlp_weights ? nullptr : lambda_in, kStepBundleNet, nullptr, *opts, R, T, W,
                   R_out, T_out, W_out, delta, lambda_out, status, 0, (cudaStream_t)stream);
}

extern "C" size_t banet_lm_step_bwd_workspace_bytes(int nb, int C, int K)
{
    if (nb <= 0 || C <= 0 || K < 0 || !lm_step_supported(6 + K, C)) return 0;
    return align_up((size_t)nb * lm_step_bwd_ws_floats(C) * sizeof(float), 256);
}

extern "C" int banet_lm_step_bwd(const float* H, const float* g, const float* rbar_sum, int nb, int N, int C, int K, const float* mlp_weights,
                                 float base, const float* lambda, const float* delta, const banet_solve_opts_t* opts, const float* R, const float* T,
                                 const float* dR_out, const float* dT_out, const float* dW_out, float* dH, float* dg, float* drbar_sum, float* dmlp,
                                 float* dlambda, float* dR, float* dT, float* dW, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    (void)base;                                                      // lambda = base ||rbar||^(2 + t) is given: its derivatives need no base
    BANET_REQUIRE(H && g && lambda && delta && opts && R && T && dR_out && dT_out && dH && dg && dlambda && dR && dT && nb > 0 && K >= 0,
                  BANET_ERR_BAD_ARG, "lm_step_bwd: bad argument");
    BANET_REQUIRE(K == 0 || (dW_out && dW), BANET_ERR_BAD_ARG, "lm_step_bwd: K=%d but dW_out / dW is null", K);
    BANET_REQUIRE(!mlp_weights || (rbar_sum && drbar_sum && dmlp && N > 0 && C > 0), BANET_ERR_BAD_ARG,
                  "lm_step_bwd: the lambda-MLP needs rbar_sum, drbar_sum, dmlp, N > 0 and C > 0");
    BANET_REQUIRE(!opts->vmatrix_batch_scramble, BANET_ERR_UNSUPPORTED, "lm_step_bwd: vmatrix_batch_scramble is not differentiated");
    BANET_REQUIRE(lm_step_supported(6 + K, mlp_weights ? C : 0), BANET_ERR_UNSUPPORTED, "lm_step_bwd: K=%d, C=%d do not fit the fused step", K, C);
    if (mlp_weights) {
        const size_t need = banet_lm_step_bwd_workspace_bytes(nb, C, K);
        BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_step_bwd: workspace %zu < %zu bytes", ws_bytes, need);
    }
    return lm_step_bwd(H, g, rbar_sum, nb, N, C, K, mlp_weights, lambda, delta, *opts, R, T, dR_out, dT_out, dW_out, 6, nullptr, dH, dg, drbar_sum,
                       dmlp, dlambda, dR, dT, dW, reinterpret_cast<float*>(ws), (cudaStream_t)stream);
}

extern "C" int banet_lm_build_bwd_weighted(const banet_level_t* lv, const float* R, const float* T, const float* W,
                                           const float* dH, const float* dg, const float* drbar_sum, int exact_sym,
                                           float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW,
                                           float* dweight, banet_stream_t stream)
{
    int rc = check_level(lv, "lm_build_bwd");
    if (rc) return rc;
    BANET_REQUIRE(R && T && dH && dg && drbar_sum && dconv1 && dconv2 && dD && dR && dT, BANET_ERR_BAD_ARG, "lm_build_bwd: null pointer");
    BANET_REQUIRE(lv->K == 0 || (W && dB && dW), BANET_ERR_BAD_ARG, "lm_build_bwd: K=%d but W / dB / dW is null", lv->K);
    return lm_build_bwd(lv, R, T, W, dH, dg, drbar_sum, exact_sym, dconv1, dconv2, dD, dB, dR, dT, dW, dweight, (cudaStream_t)stream);
}

extern "C" int banet_lm_build_bwd(const banet_level_t* lv, const float* R, const float* T, const float* W,
                                  const float* dH, const float* dg, const float* drbar_sum, int exact_sym,
                                  float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW, banet_stream_t stream)
{
    return banet_lm_build_bwd_weighted(lv, R, T, W, dH, dg, drbar_sum, exact_sym, dconv1, dconv2, dD, dB, dR, dT, dW, nullptr, stream);
}

// -------------------------------------------------------------------------------------------------
extern "C" size_t banet_lm_cost_workspace_bytes(const banet_level_t* lv)
{
    if (check_level(lv, "lm_cost_workspace_bytes") || lv->K > 256) return 0;
    return lm_cost_ws_bytes(lv);
}

extern "C" int banet_lm_cost(const banet_level_t* lv, const float* R, const float* T, const float* W, float* cost, float* nvalid, float* s,
                             float* mask, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    int rc = check_level(lv, "lm_cost");
    if (rc) return rc;
    BANET_REQUIRE(R && T && cost && nvalid, BANET_ERR_BAD_ARG, "lm_cost: null pointer");
    BANET_REQUIRE(lv->K == 0 || W, BANET_ERR_BAD_ARG, "lm_cost: K=%d but W is null", lv->K);
    BANET_REQUIRE(lv->K <= 256, BANET_ERR_UNSUPPORTED, "lm_cost: K=%d > 256 not supported", lv->K);
    const size_t need = lm_cost_ws_bytes(lv);
    BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_cost: workspace %zu < %zu bytes", ws_bytes, need);
    return lm_cost(lv, R, T, W, cost, nvalid, s, mask, ws, (cudaStream_t)stream);
}

extern "C" int banet_lm_cost_bwd(const banet_level_t* lv, const float* R, const float* T, const float* W, const float* dcost,
                                 float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW, float* dweight,
                                 banet_stream_t stream)
{
    int rc = check_level(lv, "lm_cost_bwd");
    if (rc) return rc;
    BANET_REQUIRE(R && T && dcost && dconv1 && dconv2 && dD && dR && dT, BANET_ERR_BAD_ARG, "lm_cost_bwd: null pointer");
    BANET_REQUIRE(lv->K == 0 || (W && dB && dW), BANET_ERR_BAD_ARG, "lm_cost_bwd: K=%d but W / dB / dW is null", lv->K);
    BANET_REQUIRE(lv->K <= 256, BANET_ERR_UNSUPPORTED, "lm_cost_bwd: K=%d > 256 not supported", lv->K);
    return lm_cost_bwd(lv, R, T, W, dcost, dconv1, dconv2, dD, dB, dR, dT, dW, dweight, (cudaStream_t)stream);
}

extern "C" int banet_lm_solve_update_bwd(const float* H, const float* g, const float* lambda, const float* delta, int nb, int K, const banet_solve_opts_t* opts,
                                         const float* R, const float* T, const float* dR_out, const float* dT_out, const float* dW_out,
                                         float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW, banet_stream_t stream)
{
    BANET_REQUIRE(H && g && lambda && delta && opts && R && T && dR_out && dT_out && dH && dg && dlambda && dR && dT, BANET_ERR_BAD_ARG, "lm_solve_update_bwd: null pointer");
    BANET_REQUIRE(nb > 0 && K >= 0 && (K == 0 || (dW_out && dW)), BANET_ERR_BAD_ARG, "lm_solve_update_bwd: bad shape nb=%d K=%d", nb, K);
    return lm_solve_update_bwd(H, g, lambda, delta, nb, K, *opts, R, T, dR_out, dT_out, dW_out, dH, dg, dlambda, dR, dT, dW, (cudaStream_t)stream);
}

// -------------------------------------------------------------------------------------------------
// Whole solves.  banet_lm_run (pairs), banet_lm_window_run (one dense keyframe window), banet_lm_window_batch_run (batches of windows on
// the block-arrow step) and banet_lm_keyframe_run (the keyframe layout) run one coarse-to-fine schedule, run_solve.  Each entry point
// checks its own arguments first and gives run_solve the sizes of its workspace, its size rule per level, what runs once before the
// first level and one iteration's build and step.
namespace {
int check_keyframe_level(const banet_keyframe_level_t* lv, const char* who)
{
    BANET_REQUIRE(lv, BANET_ERR_BAD_ARG, "%s: null level", who);
    BANET_REQUIRE(lv->nw > 0 && lv->nf > 0 && lv->N > 0 && lv->C > 0 && lv->K > 0 && lv->h >= 2 && lv->w >= 2, BANET_ERR_BAD_ARG,
                  "%s: bad shape nw=%d nf=%d N=%d C=%d K=%d h=%d w=%d", who, lv->nw, lv->nf, lv->N, lv->C, lv->K, lv->h, lv->w);
    BANET_REQUIRE(lv->conv2_channels == 3 * lv->C || lv->conv2_channels == lv->C, BANET_ERR_BAD_ARG,
                  "%s: conv2_channels=%d must be 3*C (reference layout) or C (F2 only)", who, lv->conv2_channels);
    BANET_REQUIRE(lv->conv1 && lv->p && lv->D && lv->B && lv->conv2 && lv->intr, BANET_ERR_BAD_ARG, "%s: null tensor", who);
    BANET_REQUIRE((long long)lv->h * lv->w * lv->conv2_channels < (1LL << 40), BANET_ERR_BAD_ARG, "%s: map too large", who);
    BANET_REQUIRE(lv->K <= 256, BANET_ERR_UNSUPPORTED, "%s: K=%d > 256 not supported", who, lv->K);
    BANET_REQUIRE(lv->C <= 2048, BANET_ERR_UNSUPPORTED, "%s: C=%d > 2048 not supported", who, lv->C);
    return BANET_OK;
}

// The keyframe build is fp32 SIMT only: AUTO resolves to it (as AUTO does wherever the tensor cores do not apply); the TF32 modes have no
// keyframe kernel.
int check_keyframe_precision(int precision, const char* who)
{
    BANET_REQUIRE(precision == BANET_PREC_AUTO || precision == BANET_PREC_FP32_SIMT || precision == BANET_PREC_TF32X1 || precision == BANET_PREC_TF32X2 ||
                  precision == BANET_PREC_TF32X3 || precision == BANET_PREC_TF32_LEVELWISE, BANET_ERR_BAD_ARG, "%s: unknown precision mode %d", who, precision);
    BANET_REQUIRE(precision == BANET_PREC_AUTO || precision == BANET_PREC_FP32_SIMT, BANET_ERR_UNSUPPORTED,
                  "%s: precision mode %d (tensor cores) has no keyframe build; use AUTO or FP32_SIMT", who, precision);
    return BANET_OK;
}

// a level of a whole solve: valid, and of level 0's batch shape
int check_run_level(const banet_level_t* levels, int l, const char* who)
{
    if (int rc = check_level(&levels[l], who)) return rc;
    BANET_REQUIRE(levels[l].nb == levels[0].nb && levels[l].K == levels[0].K, BANET_ERR_BAD_ARG, "%s: nb/K must agree across levels", who);
    return BANET_OK;
}
int check_run_level(const banet_keyframe_level_t* levels, int l, const char* who)
{
    if (int rc = check_keyframe_level(&levels[l], who)) return rc;
    BANET_REQUIRE(levels[l].nw == levels[0].nw && levels[l].nf == levels[0].nf && levels[l].K == levels[0].K, BANET_ERR_BAD_ARG,
                  "%s: nw/nf/K must agree across levels", who);
    return BANET_OK;
}

// A level's build plan.  `who` names the caller in the robust-loss and precision checks, which a workspace query reaches unchecked.
struct PairPlan : BuildPlan { int res; };                          // + the precision the level resolves to
int plan_level(const banet_level_t* lv, int precision, const char* who, PairPlan* plan)
{
    if (int rc = check_robust(lv, who)) return rc;
    plan->res = resolve_precision(lv, precision);
    return plan->res < 0 ? plan->res : plan_for(lv, plan->res, plan);
}
int plan_level(const banet_keyframe_level_t* lv, int precision, const char* who, KeyframePlan* plan)
{
    if (int rc = check_keyframe_precision(precision, who)) return rc;
    return keyframe_plan(lv, num_sms(), plan);
}
template <class Level> using PlanOf = std::conditional_t<std::is_same<Level, banet_level_t>::value, PairPlan, KeyframePlan>;

// The workspace of a whole solve: build | H | g | rbar | nvalid | lambda | delta | tail, every part but the tail 256-B aligned, for nb
// pairs of P unknowns, rbar of the widest level (maxC), and the form's lambda and delta floats and tail bytes.
struct RunSizes { size_t nb; int P, maxC; size_t lambda, delta, tail; };
struct RunCarve { size_t build, H, g, rbar, nvalid, lambda, delta, tail, total; };
struct RunWork { float *H, *g, *rbar, *nvalid, *lambda, *delta; char *build, *tail; };

template <class Level> int max_C(const Level* levels, int nlevels)
{
    int C = 0;
    for (int l = 0; l < nlevels; ++l) C = std::max(C, levels[l].C);
    return C;
}
RunSizes pair_sizes(const banet_level_t* levels, int nlevels)
{
    const int nb = levels[0].nb, P = 6 + levels[0].K;
    return {(size_t)nb, P, max_C(levels, nlevels), (size_t)nb, (size_t)nb * P, 0};
}
RunSizes window_sizes(const banet_level_t* levels, int nlevels)     // + the dense window step's matrix and factors
{
    RunSizes s = pair_sizes(levels, nlevels);
    s.tail = align_up(lm_window_step_workspace_floats(levels[0].nb, levels[0].K, s.maxC) * sizeof(float), 256);
    return s;
}
RunSizes batch_sizes(const banet_level_t* levels, int nlevels, int nw)  // + per-pair copies of W for the build + the step's per-frame factors
{
    RunSizes s = pair_sizes(levels, nlevels);
    s.tail = align_up(s.nb * levels[0].K * sizeof(float), 256) + lm_window_batch_ws_bytes(nw, levels[0].nb / nw);
    return s;
}
RunSizes keyframe_sizes(const banet_keyframe_level_t* levels, int nlevels)   // one lambda and delta [6 nf + K] per window
{
    const int nw = levels[0].nw, nf = levels[0].nf, K = levels[0].K;
    return {(size_t)nw * nf, 6 + K, max_C(levels, nlevels), (size_t)nw, (size_t)nw * (6 * nf + K), lm_window_batch_ws_bytes(nw, nf)};
}

template <class Level>
int run_carve(const Level* levels, int nlevels, int precision, const char* who, const RunSizes& s, RunCarve* c)
{
    size_t build = 0;
    for (int l = 0; l < nlevels; ++l) {
        PlanOf<Level> plan;
        if (int rc = plan_level(&levels[l], precision, who, &plan)) return rc;
        build = std::max(build, plan.ws_bytes);
    }
    size_t off = 0;
    c->build = off;  off += align_up(build, 256);
    c->H = off;      off += align_up(s.nb * s.P * s.P * 4, 256);
    c->g = off;      off += align_up(s.nb * s.P * 4, 256);
    c->rbar = off;   off += align_up(s.nb * s.maxC * 4, 256);
    c->nvalid = off; off += align_up(s.nb * 4, 256);
    c->lambda = off; off += align_up(s.lambda * 4, 256);
    c->delta = off;  off += align_up(s.delta * 4, 256);
    c->tail = off;
    c->total = off + s.tail;
    return BANET_OK;
}

__global__ void fill_kernel(float* p, int n, float v) { int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = v; }
__global__ void zero_status_kernel(int32_t* p, int n) { int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = 0; }

// The schedule of every whole solve.  Per level: its checks, the rule "lambda-MLP weights or lambda_fixed >= 0" and the form's size rule
// fits(level, use_mlp).  Then the carve, status zeroed and start(work) once.  Then per level its build plan, lambda_fixed in the first
// nlambda slots when the level has no MLP, and iters_per_level x iterate(level, plan, mlp, work): one build and one step, mlp null when
// lambda is fixed.
template <class Level, class Fits, class Start, class Iterate>
int run_solve(const char* who, const Level* levels, int nlevels, int iters_per_level, const float* const* mlp_weights, float lambda_fixed,
              int precision, const float* W, int32_t* status, void* ws, size_t ws_bytes, cudaStream_t st, const RunSizes& s, int nlambda,
              Fits fits, Start start, Iterate iterate)
{
    for (int l = 0; l < nlevels; ++l) {
        if (int rc = check_run_level(levels, l, who)) return rc;
        BANET_REQUIRE((mlp_weights && mlp_weights[l]) || lambda_fixed >= 0.f, BANET_ERR_BAD_ARG,
                      "%s: level %d has no lambda-MLP weights and lambda_fixed < 0", who, l);
        if (int rc = fits(levels[l], mlp_weights && mlp_weights[l] && lambda_fixed < 0.f)) return rc;
    }
    // a pose-only solve (K = 0) takes no W; the window forms require W with their other pointers
    BANET_REQUIRE(levels[0].K == 0 || W, BANET_ERR_BAD_ARG, "%s: K=%d but W is null", who, levels[0].K);
    RunCarve c;
    if (int rc = run_carve(levels, nlevels, precision, who, s, &c)) return rc;
    BANET_REQUIRE(ws && ws_bytes >= c.total, BANET_ERR_WORKSPACE, "%s: workspace %zu < %zu bytes", who, ws_bytes, c.total);
    char* base = reinterpret_cast<char*>(ws);
    const auto at = [base](size_t off) { return reinterpret_cast<float*>(base + off); };
    const RunWork w = {at(c.H), at(c.g), at(c.rbar), at(c.nvalid), at(c.lambda), at(c.delta), base + c.build, base + c.tail};
    const int nb = (int)s.nb;
    zero_status_kernel<<<(nb + 255) / 256, 256, 0, st>>>(status, nb);
    if (int rc = start(w)) return rc;
    for (int l = 0; l < nlevels; ++l) {
        PlanOf<Level> plan;
        if (int rc = plan_level(&levels[l], precision, who, &plan)) return rc;
        const float* mlp = mlp_weights && lambda_fixed < 0.f ? mlp_weights[l] : nullptr;
        if (!mlp) fill_kernel<<<(nlambda + 255) / 256, 256, 0, st>>>(w.lambda, nlambda, lambda_fixed);
        for (int it = 0; it < iters_per_level; ++it)
            if (int rc = iterate(levels[l], plan, mlp, w)) return rc;
    }
    BANET_CUDA_LAUNCH_CHECK(who);
    return BANET_OK;
}
}  // namespace

extern "C" size_t banet_lm_run_workspace_bytes(const banet_level_t* levels, int nlevels, int precision)
{
    RunCarve c;
    if (!levels || nlevels <= 0 || run_carve(levels, nlevels, precision, "lm_run_workspace_bytes", pair_sizes(levels, nlevels), &c)) return 0;
    return c.total;
}

extern "C" int banet_lm_run(const banet_level_t* levels, int nlevels, int iters_per_level,
                            const float* const* mlp_weights, float l2_regularizer_base, float lambda_fixed,
                            const banet_solve_opts_t* opts, int precision,
                            float* R, float* T, float* W, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(levels && nlevels > 0 && iters_per_level > 0 && opts && R && T && status, BANET_ERR_BAD_ARG, "lm_run: bad argument");
    const int nb = levels[0].nb, K = levels[0].K;
    const bool scramble = opts->vmatrix_batch_scramble != 0;
    cudaStream_t st = (cudaStream_t)stream;
    return run_solve("lm_run", levels, nlevels, iters_per_level, mlp_weights, lambda_fixed, precision, W, status, ws, ws_bytes, st,
                     pair_sizes(levels, nlevels), nb,
        [&](const banet_level_t& lv, bool use_mlp) {
            BANET_REQUIRE(lm_step_supported(6 + K, use_mlp ? lv.C : 0), BANET_ERR_UNSUPPORTED, "lm_run: K=%d, C=%d do not fit the step kernel", K, lv.C);
            return BANET_OK;
        },
        [](const RunWork&) { return BANET_OK; },
        [&](const banet_level_t& lv, const PairPlan& plan, const float* mlp, const RunWork& w) {
            int rc = build_dispatch(&lv, plan.res, plan, R, T, W, w.H, w.g, w.rbar, w.nvalid, w.build, st);
            // one launch: lambda-MLP + damping + Cholesky + update; the batch-interleaved VMatrix updates R, T after every pair's step
            if (!rc) rc = lm_step(w.H, w.g, w.rbar, nb, lv.N, lv.C, K, mlp, l2_regularizer_base, mlp ? nullptr : w.lambda, kStepBundleNet, nullptr,
                                  *opts, R, T, W, scramble ? nullptr : R, T, W, w.delta, w.lambda, status, 1, st);
            if (!rc && scramble) rc = launch_pose_update(w.delta, nb, 6 + K, 1, R, T, R, T, st);
            return rc;
        });
}

// ---- joint keyframe window (SURVEY.md section 8f-4; an extension, the reference is 2-view): nb = nf frame pairs sharing one W -------------
extern "C" size_t banet_lm_window_run_workspace_bytes(const banet_level_t* levels, int nlevels, int precision)
{
    RunCarve c;
    if (!levels || nlevels <= 0 || levels[0].K <= 0 ||
        run_carve(levels, nlevels, precision, "lm_window_run_workspace_bytes", window_sizes(levels, nlevels), &c)) return 0;
    return c.total;
}

extern "C" int banet_lm_window_run(const banet_level_t* levels, int nlevels, int iters_per_level,
                                   const float* const* mlp_weights, float l2_regularizer_base, float lambda_fixed,
                                   const banet_solve_opts_t* opts, int precision,
                                   float* R, float* T, float* W, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(levels && nlevels > 0 && iters_per_level > 0 && opts && R && T && W && status, BANET_ERR_BAD_ARG, "lm_window_run: bad argument");
    const int nf = levels[0].nb, K = levels[0].K;
    BANET_REQUIRE(K > 0 && !opts->vmatrix_batch_scramble, BANET_ERR_BAD_ARG, "lm_window_run: needs a depth basis (K > 0) and vmatrix_batch_scramble = 0");
    cudaStream_t st = (cudaStream_t)stream;
    return run_solve("lm_window_run", levels, nlevels, iters_per_level, mlp_weights, lambda_fixed, precision, W, status, ws, ws_bytes, st,
                     window_sizes(levels, nlevels), 1,
        [&](const banet_level_t& lv, bool) {
            BANET_REQUIRE(lm_window_supported(nf, K, lv.C), BANET_ERR_UNSUPPORTED, "lm_window_run: 6*%d+%d unknowns do not fit the solve kernel", nf, K);
            return BANET_OK;
        },
        [&](const RunWork&) { return lm_window_broadcast_w(W, nf, K, st); },        // frame 0's W is the window's W
        [&](const banet_level_t& lv, const PairPlan& plan, const float* mlp, const RunWork& w) {
            const int rc = build_dispatch(&lv, plan.res, plan, R, T, W, w.H, w.g, w.rbar, w.nvalid, w.build, st);
            return rc ? rc : lm_window_step(w.H, w.g, w.rbar, nf, lv.N, lv.C, K, mlp, l2_regularizer_base, mlp ? nullptr : w.lambda, *opts,
                                            R, T, W, nf, R, T, W, nullptr, reinterpret_cast<float*>(w.tail), nullptr, status, 1, st);
        });
}

extern "C" size_t banet_lm_window_solve_update_workspace_bytes(int nf, int K)
{
    if (nf <= 0 || K <= 0) return 0;
    return align_up(lm_window_step_workspace_floats(nf, K, 0) * sizeof(float), 256);
}

extern "C" int banet_lm_window_solve_update(const float* H, const float* g, const float* lambda, int nf, int K, const banet_solve_opts_t* opts,
                                            const float* R, const float* T, const float* W, float* R_out, float* T_out, float* W_out,
                                            float* delta, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(H && g && lambda && opts && R && T && W && R_out && T_out && W_out && delta && status, BANET_ERR_BAD_ARG,
                  "lm_window_solve_update: null pointer");
    BANET_REQUIRE(nf > 0 && K > 0 && !opts->vmatrix_batch_scramble, BANET_ERR_BAD_ARG,
                  "lm_window_solve_update: needs nf > 0, a depth basis (K > 0) and vmatrix_batch_scramble = 0 (nf=%d K=%d)", nf, K);
    BANET_REQUIRE(lm_window_supported(nf, K, 1), BANET_ERR_UNSUPPORTED, "lm_window_solve_update: 6*%d+%d unknowns do not fit the solve kernel", nf, K);
    const size_t need = banet_lm_window_solve_update_workspace_bytes(nf, K);
    BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_window_solve_update: workspace %zu < %zu bytes", ws_bytes, need);
    return lm_window_step(H, g, nullptr, nf, 1, 0, K, nullptr, 1.f, lambda, *opts, R, T, W, 1, R_out, T_out, W_out, delta,
                          reinterpret_cast<float*>(ws), nullptr, status, 0, (cudaStream_t)stream);
}

extern "C" size_t banet_lm_window_solve_update_bwd_workspace_bytes(int nf, int K)
{
    if (nf <= 0 || K <= 0) return 0;
    return align_up(lm_window_step_bwd_workspace_floats(nf, K) * sizeof(float), 256);
}

extern "C" int banet_lm_window_solve_update_bwd(const float* H, const float* g, const float* lambda, const float* delta, int nf, int K,
                                                const banet_solve_opts_t* opts, const float* R, const float* T,
                                                const float* dR_out, const float* dT_out, const float* dW_out,
                                                float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW,
                                                void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(H && g && lambda && delta && opts && R && T && dR_out && dT_out && dW_out && dH && dg && dlambda && dR && dT && dW, BANET_ERR_BAD_ARG,
                  "lm_window_solve_update_bwd: null pointer");
    BANET_REQUIRE(nf > 0 && K > 0 && !opts->vmatrix_batch_scramble, BANET_ERR_BAD_ARG,
                  "lm_window_solve_update_bwd: needs nf > 0, a depth basis (K > 0) and vmatrix_batch_scramble = 0 (nf=%d K=%d)", nf, K);
    BANET_REQUIRE(lm_window_supported(nf, K, 0), BANET_ERR_UNSUPPORTED, "lm_window_solve_update_bwd: 6*%d+%d unknowns do not fit the solve kernel", nf, K);
    const size_t need = banet_lm_window_solve_update_bwd_workspace_bytes(nf, K);
    BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_window_solve_update_bwd: workspace %zu < %zu bytes", ws_bytes, need);
    return lm_window_step_bwd(H, g, lambda, delta, nf, K, *opts, R, T, dR_out, dT_out, dW_out, dH, dg, dlambda, dR, dT, dW,
                              reinterpret_cast<float*>(ws), (cudaStream_t)stream);
}

// ---- batches of keyframe windows (section 3d): nb = nw nf pairs, pair w nf + f = (keyframe of window w -> frame f) -----------------------
extern "C" size_t banet_lm_window_batch_run_workspace_bytes(const banet_level_t* levels, int nlevels, int nw, int precision)
{
    RunCarve c;
    if (!levels || nlevels <= 0 || nw <= 0 || levels[0].K <= 0 || levels[0].nb % nw != 0 ||
        run_carve(levels, nlevels, precision, "lm_window_batch_run_workspace_bytes", batch_sizes(levels, nlevels, nw), &c)) return 0;
    return c.total;
}

extern "C" int banet_lm_window_batch_run(const banet_level_t* levels, int nlevels, int nw, int iters_per_level,
                                         const float* const* mlp_weights, float l2_regularizer_base, float lambda_fixed,
                                         const banet_solve_opts_t* opts, int precision,
                                         float* R, float* T, float* W, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(levels && opts && R && T && W && status, BANET_ERR_BAD_ARG, "lm_window_batch_run: null pointer");
    BANET_REQUIRE(nlevels > 0 && iters_per_level > 0 && nw > 0, BANET_ERR_BAD_ARG, "lm_window_batch_run: bad argument nlevels=%d iters=%d nw=%d",
                  nlevels, iters_per_level, nw);
    const int nb = levels[0].nb, K = levels[0].K;
    BANET_REQUIRE(K > 0 && !opts->vmatrix_batch_scramble, BANET_ERR_BAD_ARG, "lm_window_batch_run: needs a depth basis (K > 0) and vmatrix_batch_scramble = 0");
    BANET_REQUIRE(nb > 0 && nb % nw == 0, BANET_ERR_BAD_ARG, "lm_window_batch_run: nb=%d is not nw * nf with nw=%d", nb, nw);
    const int nf = nb / nw;
    cudaStream_t st = (cudaStream_t)stream;
    return run_solve("lm_window_batch_run", levels, nlevels, iters_per_level, mlp_weights, lambda_fixed, precision, W, status, ws, ws_bytes, st,
                     batch_sizes(levels, nlevels, nw), nw,
        [&](const banet_level_t& lv, bool use_mlp) {
            BANET_REQUIRE(lm_window_batch_supported(K, use_mlp ? lv.C : 0), BANET_ERR_UNSUPPORTED,
                          "lm_window_batch_run: K=%d (C=%d) does not fit the window step (K <= 256)", K, lv.C);
            return BANET_OK;
        },
        [&](const RunWork& w) { return lm_window_batch_broadcast_w(W, nw, nf, K, reinterpret_cast<float*>(w.tail), st); },
        [&](const banet_level_t& lv, const PairPlan& plan, const float* mlp, const RunWork& w) {  // one build launch and one step launch
            float* Wp = reinterpret_cast<float*>(w.tail);                   // [nb, K] per-pair copies of the windows' W
            const int rc = build_dispatch(&lv, plan.res, plan, R, T, Wp, w.H, w.g, w.rbar, w.nvalid, w.build, st);
            return rc ? rc : lm_window_batch_step(w.H, w.g, w.rbar, nw, nf, lv.N, lv.C, K, mlp, l2_regularizer_base, mlp ? nullptr : w.lambda,
                                                  *opts, R, T, W, R, T, W, Wp, w.delta, mlp ? w.lambda : nullptr, status, 1,
                                                  w.tail + align_up((size_t)nb * K * sizeof(float), 256), st);
        });
}

extern "C" size_t banet_lm_window_batch_solve_update_workspace_bytes(int nw, int nf, int K)
{
    if (nw <= 0 || nf <= 0 || K <= 0) return 0;
    return lm_window_batch_ws_bytes(nw, nf);
}

extern "C" int banet_lm_window_batch_solve_update(const float* H, const float* g, const float* lambda, int nw, int nf, int K, const banet_solve_opts_t* opts,
                                                  const float* R, const float* T, const float* W, float* R_out, float* T_out, float* W_out,
                                                  float* delta, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(H && g && lambda && opts && R && T && W && R_out && T_out && W_out && delta && status, BANET_ERR_BAD_ARG,
                  "lm_window_batch_solve_update: null pointer");
    BANET_REQUIRE(nw > 0 && nf > 0 && K > 0 && !opts->vmatrix_batch_scramble, BANET_ERR_BAD_ARG,
                  "lm_window_batch_solve_update: needs nw, nf > 0, a depth basis (K > 0) and vmatrix_batch_scramble = 0 (nw=%d nf=%d K=%d)", nw, nf, K);
    BANET_REQUIRE(lm_window_batch_supported(K, 0), BANET_ERR_UNSUPPORTED, "lm_window_batch_solve_update: K=%d does not fit the window step (K <= 256)", K);
    const size_t need = banet_lm_window_batch_solve_update_workspace_bytes(nw, nf, K);
    BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_window_batch_solve_update: workspace %zu < %zu bytes", ws_bytes, need);
    return lm_window_batch_step(H, g, nullptr, nw, nf, 1, 0, K, nullptr, 1.f, lambda, *opts, R, T, W, R_out, T_out, W_out, nullptr, delta,
                                nullptr, status, 0, ws, (cudaStream_t)stream);
}

extern "C" size_t banet_lm_window_batch_solve_update_bwd_workspace_bytes(int nw, int nf, int K)
{
    if (nw <= 0 || nf <= 0 || K <= 0) return 0;
    return lm_window_batch_ws_bytes(nw, nf);
}

extern "C" int banet_lm_window_batch_solve_update_bwd(const float* H, const float* g, const float* lambda, const float* delta, int nw, int nf, int K,
                                                      const banet_solve_opts_t* opts, const float* R, const float* T,
                                                      const float* dR_out, const float* dT_out, const float* dW_out,
                                                      float* dH, float* dg, float* dlambda, float* dR, float* dT, float* dW,
                                                      void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(H && g && lambda && delta && opts && R && T && dR_out && dT_out && dW_out && dH && dg && dlambda && dR && dT && dW, BANET_ERR_BAD_ARG,
                  "lm_window_batch_solve_update_bwd: null pointer");
    BANET_REQUIRE(nw > 0 && nf > 0 && K > 0 && !opts->vmatrix_batch_scramble, BANET_ERR_BAD_ARG,
                  "lm_window_batch_solve_update_bwd: needs nw, nf > 0, a depth basis (K > 0) and vmatrix_batch_scramble = 0 (nw=%d nf=%d K=%d)", nw, nf, K);
    BANET_REQUIRE(lm_window_batch_supported(K, 0), BANET_ERR_UNSUPPORTED, "lm_window_batch_solve_update_bwd: K=%d does not fit the window step (K <= 256)", K);
    const size_t need = banet_lm_window_batch_solve_update_bwd_workspace_bytes(nw, nf, K);
    BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_window_batch_solve_update_bwd: workspace %zu < %zu bytes", ws_bytes, need);
    return lm_window_batch_step_bwd(H, g, lambda, delta, nw, nf, K, *opts, R, T, dR_out, dT_out, dW_out, dH, dg, dlambda, dR, dT, dW, ws, (cudaStream_t)stream);
}

// ---- keyframe-layout window batches (section 3e): the keyframe tensors once per window ------------------------------------------------
extern "C" size_t banet_lm_keyframe_build_workspace_bytes(const banet_keyframe_level_t* lv)
{
    if (check_keyframe_level(lv, "lm_keyframe_build")) return 0;
    KeyframePlan plan;
    if (keyframe_plan(lv, num_sms(), &plan) != BANET_OK) return 0;
    return plan.ws_bytes;
}

extern "C" int banet_lm_keyframe_build(const banet_keyframe_level_t* lv, const float* R, const float* T, const float* W,
                                       float* H, float* g, float* rbar_sum, float* nvalid, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    int rc = check_keyframe_level(lv, "lm_keyframe_build");
    if (rc) return rc;
    BANET_REQUIRE(R && T && W && H && g && rbar_sum && nvalid, BANET_ERR_BAD_ARG, "lm_keyframe_build: null pointer");
    KeyframePlan plan;
    rc = keyframe_plan(lv, num_sms(), &plan);
    if (rc) return rc;
    BANET_REQUIRE(ws && ws_bytes >= plan.ws_bytes, BANET_ERR_WORKSPACE, "lm_keyframe_build: workspace %zu < %zu bytes", ws_bytes, plan.ws_bytes);
    return keyframe_build(lv, plan, R, T, W, H, g, rbar_sum, nvalid, ws, (cudaStream_t)stream);
}

extern "C" int banet_lm_keyframe_build_bwd_weighted(const banet_keyframe_level_t* lv, const float* R, const float* T, const float* W,
                                                    const float* dH, const float* dg, const float* drbar_sum, int exact_sym,
                                                    float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW,
                                                    float* dweight, banet_stream_t stream)
{
    int rc = check_keyframe_level(lv, "lm_keyframe_build_bwd");
    if (rc) return rc;
    BANET_REQUIRE(R && T && W && dH && dg && drbar_sum && dconv1 && dconv2 && dD && dB && dR && dT && dW, BANET_ERR_BAD_ARG,
                  "lm_keyframe_build_bwd: null pointer");
    BANET_REQUIRE(lv->conv2_channels == 3 * lv->C, BANET_ERR_UNSUPPORTED, "lm_keyframe_build_bwd: conv2 must be the [F2|gx|gy] (3C) layout");
    BANET_REQUIRE(keyframe_build_bwd_supported(lv->nf, lv->K, lv->C), BANET_ERR_UNSUPPORTED,
                  "lm_keyframe_build_bwd: K=%d, C=%d do not fit shared memory", lv->K, lv->C);
    return keyframe_build_bwd(lv, R, T, W, dH, dg, drbar_sum, exact_sym, dconv1, dconv2, dD, dB, dR, dT, dW, dweight, (cudaStream_t)stream);
}

extern "C" int banet_lm_keyframe_build_bwd(const banet_keyframe_level_t* lv, const float* R, const float* T, const float* W,
                                           const float* dH, const float* dg, const float* drbar_sum, int exact_sym,
                                           float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW, banet_stream_t stream)
{
    return banet_lm_keyframe_build_bwd_weighted(lv, R, T, W, dH, dg, drbar_sum, exact_sym, dconv1, dconv2, dD, dB, dR, dT, dW, nullptr, stream);
}

extern "C" size_t banet_lm_keyframe_cost_workspace_bytes(const banet_keyframe_level_t* lv)
{
    if (check_keyframe_level(lv, "lm_keyframe_cost_workspace_bytes")) return 0;
    return keyframe_cost_ws_bytes(lv);
}

extern "C" int banet_lm_keyframe_cost(const banet_keyframe_level_t* lv, const float* R, const float* T, const float* W, float* cost, float* nvalid,
                                      float* s, float* mask, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    int rc = check_keyframe_level(lv, "lm_keyframe_cost");
    if (rc) return rc;
    BANET_REQUIRE(R && T && W && cost && nvalid, BANET_ERR_BAD_ARG, "lm_keyframe_cost: null pointer");
    const size_t need = keyframe_cost_ws_bytes(lv);
    BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_keyframe_cost: workspace %zu < %zu bytes", ws_bytes, need);
    return keyframe_cost(lv, R, T, W, cost, nvalid, s, mask, ws, (cudaStream_t)stream);
}

extern "C" int banet_lm_keyframe_cost_bwd(const banet_keyframe_level_t* lv, const float* R, const float* T, const float* W, const float* dcost,
                                          float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW, float* dweight,
                                          banet_stream_t stream)
{
    int rc = check_keyframe_level(lv, "lm_keyframe_cost_bwd");
    if (rc) return rc;
    BANET_REQUIRE(R && T && W && dcost && dconv1 && dconv2 && dD && dB && dR && dT && dW, BANET_ERR_BAD_ARG, "lm_keyframe_cost_bwd: null pointer");
    return keyframe_cost_bwd(lv, R, T, W, dcost, dconv1, dconv2, dD, dB, dR, dT, dW, dweight, (cudaStream_t)stream);
}

extern "C" size_t banet_lm_keyframe_run_workspace_bytes(const banet_keyframe_level_t* levels, int nlevels, int precision)
{
    if (!levels || nlevels <= 0 || check_keyframe_precision(precision, "lm_keyframe_run")) return 0;
    for (int l = 0; l < nlevels; ++l)
        if (check_keyframe_level(&levels[l], "lm_keyframe_run") || levels[l].nw != levels[0].nw || levels[l].nf != levels[0].nf ||
            levels[l].K != levels[0].K) return 0;
    RunCarve c;
    return run_carve(levels, nlevels, precision, "lm_keyframe_run", keyframe_sizes(levels, nlevels), &c) ? 0 : c.total;
}

extern "C" int banet_lm_keyframe_run(const banet_keyframe_level_t* levels, int nlevels, int iters_per_level,
                                     const float* const* mlp_weights, float l2_regularizer_base, float lambda_fixed,
                                     const banet_solve_opts_t* opts, int precision,
                                     float* R, float* T, float* W, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(levels && opts && R && T && W && status, BANET_ERR_BAD_ARG, "lm_keyframe_run: null pointer");
    BANET_REQUIRE(nlevels > 0 && iters_per_level > 0, BANET_ERR_BAD_ARG, "lm_keyframe_run: bad argument nlevels=%d iters=%d", nlevels, iters_per_level);
    BANET_REQUIRE(!opts->vmatrix_batch_scramble, BANET_ERR_BAD_ARG, "lm_keyframe_run: needs vmatrix_batch_scramble = 0");
    const int nw = levels[0].nw, nf = levels[0].nf, K = levels[0].K;
    cudaStream_t st = (cudaStream_t)stream;
    return run_solve("lm_keyframe_run", levels, nlevels, iters_per_level, mlp_weights, lambda_fixed, precision, W, status, ws, ws_bytes, st,
                     keyframe_sizes(levels, nlevels), nw,
        [&](const banet_keyframe_level_t& lv, bool use_mlp) {
            BANET_REQUIRE(lm_window_batch_supported(K, use_mlp ? lv.C : 0), BANET_ERR_UNSUPPORTED,
                          "lm_keyframe_run: K=%d (C=%d) does not fit the window step", K, lv.C);
            return BANET_OK;
        },
        [](const RunWork&) { return BANET_OK; },
        [&](const banet_keyframe_level_t& lv, const KeyframePlan& plan, const float* mlp, const RunWork& w) {  // one build and one step launch
            const int rc = keyframe_build(&lv, plan, R, T, W, w.H, w.g, w.rbar, w.nvalid, w.build, st);
            return rc ? rc : lm_window_batch_step(w.H, w.g, w.rbar, nw, nf, lv.N, lv.C, K, mlp, l2_regularizer_base, mlp ? nullptr : w.lambda,
                                                  *opts, R, T, W, R, T, W, nullptr, w.delta, mlp ? w.lambda : nullptr, status, 1, w.tail, st);
        });
}

extern "C" size_t banet_lm_track_legacy_workspace_bytes(const banet_level_t* levels, int nlevels)
{
    if (!levels || nlevels <= 0) return 0;
    for (int l = 0; l < nlevels; ++l) if (check_level(&levels[l], "lm_track_legacy") || levels[l].K != 0) return 0;
    return lm_track_legacy_workspace_bytes(levels, nlevels);
}

extern "C" int banet_lm_track_legacy(const banet_level_t* levels, int nlevels, const int* level_iters, const float* const* mlp_weights,
                                     const banet_legacy_opts_t* opts, float* R, float* T, int32_t* iters_done, float* valid_ratio, int32_t* status,
                                     void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(levels && nlevels > 0 && level_iters && opts && R && T && valid_ratio && status, BANET_ERR_BAD_ARG, "lm_track_legacy: bad argument");
    for (int l = 0; l < nlevels; ++l) {
        int rc = check_level(&levels[l], "lm_track_legacy");
        if (rc) return rc;
        BANET_REQUIRE(levels[l].feature_dtype == BANET_DTYPE_F32, BANET_ERR_UNSUPPORTED,
                      "lm_track_legacy: level %d has bf16 features; the legacy tracker takes fp32 features only", l);
        BANET_REQUIRE(!levels[l].weight, BANET_ERR_UNSUPPORTED,
                      "lm_track_legacy: level %d has point weights; the tracker's accept / reject test re-evaluates an unweighted residual", l);
        BANET_REQUIRE(levels[l].robust == BANET_ROBUST_NONE, BANET_ERR_UNSUPPORTED,
                      "lm_track_legacy: level %d has a robust loss; the tracker's accept / reject test re-evaluates the plain residual", l);
        BANET_REQUIRE(levels[l].K == 0 && levels[l].nb == levels[0].nb && levels[l].conv2_channels == 3 * levels[l].C && level_iters[l] >= 0, BANET_ERR_BAD_ARG,
                      "lm_track_legacy: level %d must be pose-only (K=0) with the [F2|gx|gy] layout and the same batch size", l);
    }
    return lm_track_legacy(levels, nlevels, level_iters, mlp_weights, *opts, R, T, iters_done, valid_ratio, status, ws, ws_bytes, (cudaStream_t)stream);
}
