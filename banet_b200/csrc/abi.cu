// extern "C" entry points of libbanet.so (see include/banet_abi.h) + the LM driver loop.
#include "common.cuh"
#include "lm_build.h"
#include <string.h>

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

static int check_level(const banet_level_t* lv, const char* who)
{
    BANET_REQUIRE(lv, BANET_ERR_BAD_ARG, "%s: null level", who);
    BANET_REQUIRE(lv->nb > 0 && lv->N > 0 && lv->C > 0 && lv->K >= 0 && lv->h >= 2 && lv->w >= 2, BANET_ERR_BAD_ARG,
                  "%s: bad shape nb=%d N=%d C=%d K=%d h=%d w=%d", who, lv->nb, lv->N, lv->C, lv->K, lv->h, lv->w);
    BANET_REQUIRE(lv->conv2_channels == 3 * lv->C || lv->conv2_channels == lv->C, BANET_ERR_BAD_ARG,
                  "%s: conv2_channels=%d must be 3*C (reference layout) or C (F2 only)", who, lv->conv2_channels);
    BANET_REQUIRE(lv->conv1 && lv->conv2 && lv->intr && lv->p && lv->D, BANET_ERR_BAD_ARG, "%s: null tensor", who);
    BANET_REQUIRE(lv->K == 0 || lv->B, BANET_ERR_BAD_ARG, "%s: K=%d but B is null", who, lv->K);
    BANET_REQUIRE((long long)lv->h * lv->w * lv->conv2_channels < (1LL << 40), BANET_ERR_BAD_ARG, "%s: map too large", who);
    BANET_REQUIRE((lv->grid_w == 0 && lv->grid_h == 0) || (lv->grid_w > 0 && lv->grid_h > 0 && (long long)lv->grid_w * lv->grid_h == lv->N),
                  BANET_ERR_BAD_ARG, "%s: grid %dx%d does not match N=%d", who, lv->grid_w, lv->grid_h, lv->N);
    return BANET_OK;
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
    const banet_tuning_t def = {0, 0, 4, 0, 0, 0};
    if (!t) { set_tuning(def); return BANET_OK; }
    BANET_REQUIRE((t->tc_generation == 0 || t->tc_generation == 6 || t->tc_generation == 7) && t->tc7_band_rows >= 1 &&
                  t->tc6_band_rows >= 0 && t->tc6_l2_hints >= 0 && t->tc6_l2_hints <= 3 && t->tc6_tap_prefetch >= 0 && t->tc6_tap_prefetch <= 3, BANET_ERR_BAD_ARG,
                  "set_tuning: tc_generation must be 0, 6 or 7, tc7_band_rows >= 1, tc6_band_rows >= 0, tc6_l2_hints and tc6_tap_prefetch in 0..3");
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
    if (!lv) return 0;
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

extern "C" int banet_lm_build_bwd(const banet_level_t* lv, const float* R, const float* T, const float* W,
                                  const float* dH, const float* dg, const float* drbar_sum, int exact_sym,
                                  float* dconv1, float* dconv2, float* dD, float* dB, float* dR, float* dT, float* dW, banet_stream_t stream)
{
    int rc = check_level(lv, "lm_build_bwd");
    if (rc) return rc;
    BANET_REQUIRE(R && T && dH && dg && drbar_sum && dconv1 && dconv2 && dD && dR && dT, BANET_ERR_BAD_ARG, "lm_build_bwd: null pointer");
    BANET_REQUIRE(lv->K == 0 || (W && dB && dW), BANET_ERR_BAD_ARG, "lm_build_bwd: K=%d but W / dB / dW is null", lv->K);
    return lm_build_bwd(lv, R, T, W, dH, dg, drbar_sum, exact_sym, dconv1, dconv2, dD, dB, dR, dT, dW, (cudaStream_t)stream);
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
// whole solve
namespace {
struct RunCarve { size_t build, H, g, rbar, nvalid, lambda, delta, total; };
int carve(const banet_level_t* levels, int nlevels, int precision, RunCarve* c)
{
    size_t build = 0; int maxC = 0;
    const int nb = levels[0].nb, K = levels[0].K, P = 6 + K;
    for (int l = 0; l < nlevels; ++l) {
        BuildPlan plan;
        const int res = resolve_precision(&levels[l], precision);
        if (res < 0) return res;
        int rc = plan_for(&levels[l], res, &plan);
        if (rc) return rc;
        if (plan.ws_bytes > build) build = plan.ws_bytes;
        if (levels[l].C > maxC) maxC = levels[l].C;
    }
    size_t off = 0;
    c->build = off;  off += align_up(build, 256);
    c->H = off;      off += align_up((size_t)nb * P * P * 4, 256);
    c->g = off;      off += align_up((size_t)nb * P * 4, 256);
    c->rbar = off;   off += align_up((size_t)nb * maxC * 4, 256);
    c->nvalid = off; off += align_up((size_t)nb * 4, 256);
    c->lambda = off; off += align_up((size_t)nb * 4, 256);
    c->delta = off;  off += align_up((size_t)nb * P * 4, 256);
    c->total = off;
    return BANET_OK;
}
__global__ void fill_kernel(float* p, int n, float v) { int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = v; }
__global__ void zero_status_kernel(int32_t* p, int n) { int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = 0; }
}  // namespace

extern "C" size_t banet_lm_run_workspace_bytes(const banet_level_t* levels, int nlevels, int precision)
{
    if (!levels || nlevels <= 0) return 0;
    RunCarve c;
    if (carve(levels, nlevels, precision, &c) != BANET_OK) return 0;
    return c.total;
}

extern "C" int banet_lm_run(const banet_level_t* levels, int nlevels, int iters_per_level,
                            const float* const* mlp_weights, float l2_regularizer_base, float lambda_fixed,
                            const banet_solve_opts_t* opts, int precision,
                            float* R, float* T, float* W, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(levels && nlevels > 0 && iters_per_level > 0 && opts && R && T && status, BANET_ERR_BAD_ARG, "lm_run: bad argument");
    const int nb = levels[0].nb, K = levels[0].K;
    for (int l = 0; l < nlevels; ++l) {
        int rc = check_level(&levels[l], "lm_run");
        if (rc) return rc;
        BANET_REQUIRE(levels[l].nb == nb && levels[l].K == K, BANET_ERR_BAD_ARG, "lm_run: nb/K must agree across levels");
        BANET_REQUIRE((mlp_weights && mlp_weights[l]) || lambda_fixed >= 0.f, BANET_ERR_BAD_ARG,
                      "lm_run: level %d has no lambda-MLP weights and lambda_fixed < 0", l);
    }
    BANET_REQUIRE(K == 0 || W, BANET_ERR_BAD_ARG, "lm_run: K=%d but W is null", K);
    RunCarve c;
    int rc = carve(levels, nlevels, precision, &c);
    if (rc) return rc;
    BANET_REQUIRE(ws && ws_bytes >= c.total, BANET_ERR_WORKSPACE, "lm_run: workspace %zu < %zu bytes", ws_bytes, c.total);
    cudaStream_t st = (cudaStream_t)stream;
    char* base = reinterpret_cast<char*>(ws);
    float* H = reinterpret_cast<float*>(base + c.H);
    float* g = reinterpret_cast<float*>(base + c.g);
    float* rbar = reinterpret_cast<float*>(base + c.rbar);
    float* nvalid = reinterpret_cast<float*>(base + c.nvalid);
    float* lam = reinterpret_cast<float*>(base + c.lambda);
    float* delta = reinterpret_cast<float*>(base + c.delta);
    zero_status_kernel<<<(nb + 255) / 256, 256, 0, st>>>(status, nb);
    for (int l = 0; l < nlevels; ++l) {
        const banet_level_t* lv = &levels[l];
        BuildPlan plan;
        const int res = resolve_precision(lv, precision);
        if (res < 0) return res;
        rc = plan_for(lv, res, &plan);
        if (rc) return rc;
        const bool use_mlp = mlp_weights && mlp_weights[l] && lambda_fixed < 0.f;
        if (!use_mlp) fill_kernel<<<(nb + 255) / 256, 256, 0, st>>>(lam, nb, lambda_fixed);
        for (int it = 0; it < iters_per_level; ++it) {
            rc = build_dispatch(lv, res, plan, R, T, W, H, g, rbar, nvalid, base + c.build, st);
            if (rc) return rc;
            const int P = 6 + K;
            if (!opts->vmatrix_batch_scramble && lm_step_supported(P, lv->C)) {      // one launch: lambda-MLP + damping + Cholesky + update
                rc = lm_step(H, g, rbar, nb, lv->N, lv->C, K, use_mlp ? mlp_weights[l] : nullptr, l2_regularizer_base, use_mlp ? nullptr : lam,
                             kStepBundleNet, nullptr, *opts, R, T, W, R, T, W, delta, lam, status, 1, st);
                if (rc) return rc;
                continue;
            }
            if (use_mlp) {
                rc = lm_lambda(rbar, nb, lv->N, lv->C, mlp_weights[l], l2_regularizer_base, lam, st);
                if (rc) return rc;
            }
            rc = lm_solve_update(H, g, lam, nb, K, *opts, R, T, W, R, T, W, delta, status, 1, st);
            if (rc) return rc;
        }
    }
    BANET_CUDA_LAUNCH_CHECK("lm_run");
    return BANET_OK;
}

// ---- joint keyframe window (SURVEY.md section 8f-4; an extension, the reference is 2-view): nb = nf frame pairs sharing one W -------------
extern "C" size_t banet_lm_window_run_workspace_bytes(const banet_level_t* levels, int nlevels, int precision)
{
    if (!levels || nlevels <= 0 || levels[0].K <= 0) return 0;
    RunCarve c;
    if (carve(levels, nlevels, precision, &c) != BANET_OK) return 0;
    int maxC = 0;
    for (int l = 0; l < nlevels; ++l) if (levels[l].C > maxC) maxC = levels[l].C;
    return c.total + align_up(lm_window_step_workspace_floats(levels[0].nb, levels[0].K, maxC) * sizeof(float), 256);
}

extern "C" int banet_lm_window_run(const banet_level_t* levels, int nlevels, int iters_per_level,
                                   const float* const* mlp_weights, float l2_regularizer_base, float lambda_fixed,
                                   const banet_solve_opts_t* opts, int precision,
                                   float* R, float* T, float* W, int32_t* status, void* ws, size_t ws_bytes, banet_stream_t stream)
{
    BANET_REQUIRE(levels && nlevels > 0 && iters_per_level > 0 && opts && R && T && W && status, BANET_ERR_BAD_ARG, "lm_window_run: bad argument");
    const int nf = levels[0].nb, K = levels[0].K;
    BANET_REQUIRE(K > 0 && !opts->vmatrix_batch_scramble, BANET_ERR_BAD_ARG, "lm_window_run: needs a depth basis (K > 0) and vmatrix_batch_scramble = 0");
    int maxC = 0;
    for (int l = 0; l < nlevels; ++l) {
        int rc = check_level(&levels[l], "lm_window_run");
        if (rc) return rc;
        BANET_REQUIRE(levels[l].nb == nf && levels[l].K == K, BANET_ERR_BAD_ARG, "lm_window_run: nb/K must agree across levels");
        BANET_REQUIRE((mlp_weights && mlp_weights[l]) || lambda_fixed >= 0.f, BANET_ERR_BAD_ARG,
                      "lm_window_run: level %d has no lambda-MLP weights and lambda_fixed < 0", l);
        BANET_REQUIRE(lm_window_supported(nf, K, levels[l].C), BANET_ERR_UNSUPPORTED, "lm_window_run: 6*%d+%d unknowns do not fit the solve kernel", nf, K);
        if (levels[l].C > maxC) maxC = levels[l].C;
    }
    RunCarve c;
    int rc = carve(levels, nlevels, precision, &c);
    if (rc) return rc;
    const size_t need = c.total + align_up(lm_window_step_workspace_floats(nf, K, maxC) * sizeof(float), 256);
    BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_window_run: workspace %zu < %zu bytes", ws_bytes, need);
    cudaStream_t st = (cudaStream_t)stream;
    char* base = reinterpret_cast<char*>(ws);
    float* H = reinterpret_cast<float*>(base + c.H);
    float* g = reinterpret_cast<float*>(base + c.g);
    float* rbar = reinterpret_cast<float*>(base + c.rbar);
    float* nvalid = reinterpret_cast<float*>(base + c.nvalid);
    float* lam = reinterpret_cast<float*>(base + c.lambda);
    float* wsw = reinterpret_cast<float*>(base + c.total);
    zero_status_kernel<<<(nf + 255) / 256, 256, 0, st>>>(status, nf);
    rc = lm_window_broadcast_w(W, nf, K, st);                      // frame 0's W is the window's W
    if (rc) return rc;
    for (int l = 0; l < nlevels; ++l) {
        const banet_level_t* lv = &levels[l];
        BuildPlan plan;
        const int res = resolve_precision(lv, precision);
        if (res < 0) return res;
        rc = plan_for(lv, res, &plan);
        if (rc) return rc;
        const bool use_mlp = mlp_weights && mlp_weights[l] && lambda_fixed < 0.f;
        if (!use_mlp) fill_kernel<<<1, 32, 0, st>>>(lam, 1, lambda_fixed);
        for (int it = 0; it < iters_per_level; ++it) {
            rc = build_dispatch(lv, res, plan, R, T, W, H, g, rbar, nvalid, base + c.build, st);
            if (rc) return rc;
            rc = lm_window_step(H, g, rbar, nf, lv->N, lv->C, K, use_mlp ? mlp_weights[l] : nullptr, l2_regularizer_base, use_mlp ? nullptr : lam,
                                *opts, R, T, W, nf, R, T, W, nullptr, wsw, nullptr, status, 1, st);
            if (rc) return rc;
        }
    }
    BANET_CUDA_LAUNCH_CHECK("lm_window_run");
    return BANET_OK;
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
    BANET_REQUIRE(lm_window_supported(nf, K, 1) && solve_bwd_supported(6 * nf + K), BANET_ERR_UNSUPPORTED,
                  "lm_window_solve_update_bwd: 6*%d+%d unknowns do not fit the solve kernels", nf, K);
    const size_t need = banet_lm_window_solve_update_bwd_workspace_bytes(nf, K);
    BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_window_solve_update_bwd: workspace %zu < %zu bytes", ws_bytes, need);
    return lm_window_step_bwd(H, g, lambda, delta, nf, K, *opts, R, T, dR_out, dT_out, dW_out, dH, dg, dlambda, dR, dT, dW,
                              reinterpret_cast<float*>(ws), (cudaStream_t)stream);
}

// ---- batches of keyframe windows (section 3d): nb = nw nf pairs, pair w nf + f = (keyframe of window w -> frame f) -----------------------
namespace {
size_t batch_run_extra(int nw, int nf, int K)                     // per-pair copies of W for the build + the step's per-frame factors
{
    return align_up((size_t)nw * nf * K * sizeof(float), 256) + lm_window_batch_ws_bytes(nw, nf);
}
}  // namespace

extern "C" size_t banet_lm_window_batch_run_workspace_bytes(const banet_level_t* levels, int nlevels, int nw, int precision)
{
    if (!levels || nlevels <= 0 || nw <= 0 || levels[0].K <= 0 || levels[0].nb % nw != 0) return 0;
    RunCarve c;
    if (carve(levels, nlevels, precision, &c) != BANET_OK) return 0;
    return c.total + batch_run_extra(nw, levels[0].nb / nw, levels[0].K);
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
    for (int l = 0; l < nlevels; ++l) {
        int rc = check_level(&levels[l], "lm_window_batch_run");
        if (rc) return rc;
        BANET_REQUIRE(levels[l].nb == nb && levels[l].K == K, BANET_ERR_BAD_ARG, "lm_window_batch_run: nb/K must agree across levels");
        BANET_REQUIRE((mlp_weights && mlp_weights[l]) || lambda_fixed >= 0.f, BANET_ERR_BAD_ARG,
                      "lm_window_batch_run: level %d has no lambda-MLP weights and lambda_fixed < 0", l);
        const bool use_mlp = mlp_weights && mlp_weights[l] && lambda_fixed < 0.f;
        BANET_REQUIRE(lm_window_batch_supported(K, use_mlp ? levels[l].C : 0), BANET_ERR_UNSUPPORTED,
                      "lm_window_batch_run: K=%d (C=%d) does not fit the window step (K <= 256)", K, levels[l].C);
    }
    RunCarve c;
    int rc = carve(levels, nlevels, precision, &c);
    if (rc) return rc;
    const size_t need = c.total + batch_run_extra(nw, nf, K);
    BANET_REQUIRE(ws && ws_bytes >= need, BANET_ERR_WORKSPACE, "lm_window_batch_run: workspace %zu < %zu bytes", ws_bytes, need);
    cudaStream_t st = (cudaStream_t)stream;
    char* base = reinterpret_cast<char*>(ws);
    float* H = reinterpret_cast<float*>(base + c.H);
    float* g = reinterpret_cast<float*>(base + c.g);
    float* rbar = reinterpret_cast<float*>(base + c.rbar);
    float* nvalid = reinterpret_cast<float*>(base + c.nvalid);
    float* lam = reinterpret_cast<float*>(base + c.lambda);            // [nw]
    float* delta = reinterpret_cast<float*>(base + c.delta);          // [nw, 6 nf + K] <= [nb, 6 + K]
    float* Wp = reinterpret_cast<float*>(base + c.total);             // [nb, K] per-pair copies of the windows' W
    void* fws = base + c.total + align_up((size_t)nb * K * sizeof(float), 256);
    zero_status_kernel<<<(nb + 255) / 256, 256, 0, st>>>(status, nb);
    rc = lm_window_batch_broadcast_w(W, nw, nf, K, Wp, st);
    if (rc) return rc;
    for (int l = 0; l < nlevels; ++l) {
        const banet_level_t* lv = &levels[l];
        BuildPlan plan;
        const int res = resolve_precision(lv, precision);
        if (res < 0) return res;
        rc = plan_for(lv, res, &plan);
        if (rc) return rc;
        const bool use_mlp = mlp_weights && mlp_weights[l] && lambda_fixed < 0.f;
        if (!use_mlp) fill_kernel<<<(nw + 255) / 256, 256, 0, st>>>(lam, nw, lambda_fixed);
        for (int it = 0; it < iters_per_level; ++it) {                // one build launch and one step launch per iteration
            rc = build_dispatch(lv, res, plan, R, T, Wp, H, g, rbar, nvalid, base + c.build, st);
            if (rc) return rc;
            rc = lm_window_batch_step(H, g, rbar, nw, nf, lv->N, lv->C, K, use_mlp ? mlp_weights[l] : nullptr, l2_regularizer_base,
                                      use_mlp ? nullptr : lam, *opts, R, T, W, R, T, W, Wp, delta, use_mlp ? lam : nullptr, status, 1, fws, st);
            if (rc) return rc;
        }
    }
    BANET_CUDA_LAUNCH_CHECK("lm_window_batch_run");
    return BANET_OK;
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
        BANET_REQUIRE(levels[l].K == 0 && levels[l].nb == levels[0].nb && levels[l].conv2_channels == 3 * levels[l].C && level_iters[l] >= 0, BANET_ERR_BAD_ARG,
                      "lm_track_legacy: level %d must be pose-only (K=0) with the [F2|gx|gy] layout and the same batch size", l);
    }
    return lm_track_legacy(levels, nlevels, level_iters, mlp_weights, *opts, R, T, iters_done, valid_ratio, status, ws, ws_bytes, (cudaStream_t)stream);
}
