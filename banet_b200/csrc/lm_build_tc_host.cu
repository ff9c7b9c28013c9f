// Host side of the tensor-core build path (sm_90a: TMA + mbarrier pipelines + warp-level tf32 MMA): support check, launch plan,
// tensor map, dispatch.
//
// Maths and partial-slot contract are those of lm_build.cu (reference bundlenet.py:206-263 + utils.cu:219-417); the basis contraction
// runs on the tensor cores:
//
//     D[128 x 136] += Bt^T R          per 64-pixel tile, tf32 mma.sync, fp32 accumulate in registers
//        Bt [64 px x 128]  the basis tile exactly as it lies in HBM (TMA, 128B/32B-atom swizzle)
//        R  [64 px x 160]  row n = [ s_n * b_n (128) | v_n (6) | t_n | 0 ... ]  built by the algebra warps, same layout
//     => D[i][j<128] = H_dd[i][j],  D[i][128+r] = H_cd[r][i] (r<6),  D[i][134] = g_d[i]
//
// Precision modes (tf32 keeps 10 mantissa bits; products are exact, accumulation is fp32):
//   MODE 1  one pass:   A and R both rounded by us (A stochastically, in place; R to nearest)
//   MODE 2  two passes: + A_lo = b - trunc(b)                       (only R's unbiased rounding remains)
//   MODE 3  three passes: + R_lo = s*b - rna(s*b)                   (fp32-grade: the dropped term is ~2^-22)
//
// Tiles: 64 points.  With the dense-grid hint (banet_level_t::grid_w/h) a tile is an 8x8 pixel patch fetched by ONE 3-D TMA box;
// without the hint a tile is 64 consecutive points (2-D TMA box).
//
// Kernel: generation 6 (lm_build_tc6.cu) covers everything (both conv2 layouts, dense grids and point lists, every mode, fp32 and bf16
// features, fp32 and bf16 bases): taps by ld.global.
#include "common.cuh"
#include "lm_build.h"
#include "tc_utils.cuh"
#include "tmap.h"

namespace banet {

constexpr int TC_TILE = 64;

int lm_build_tc6_launch(int mode, bool fly, int nch, int kblk, bool is_bf16, bool basis_bf16, const CUtensorMap& tm, const BuildParams& prm, int grid,
                        cudaStream_t st);

constexpr int kTc6DefaultBandRows = 1, kTc6DefaultL2Hints = 0, kTc6DefaultTapPrefetch = 0;
static banet_tuning_t g_tuning = {0, 0, 0};
void set_tuning(const banet_tuning_t& t) { g_tuning = t; }
const banet_tuning_t& tuning() { return g_tuning; }

// The F2-only gather packs the four tap columns of a pixel into 16 bits each (lm_build_tc6.cu, the geometry warps' cx[]), so that
// layout needs w < 65536; a wider map resolves to the SIMT kernel under AUTO and is BANET_ERR_UNSUPPORTED in an explicit TF32 mode.
static bool tc_f2_width_ok(const banet_level_t* lv) { return lv->conv2_channels != lv->C || lv->w < 65536; }

bool tc_supported(const banet_level_t* lv)
{
    const bool k_ok = lv->K == 128 || lv->K == 64 || lv->K == 32;
    return k_ok && (lv->C == 64 || lv->C == 128) && (lv->conv2_channels == lv->C || lv->conv2_channels == 3 * lv->C) &&
           ((reinterpret_cast<uintptr_t>(lv->conv1) | reinterpret_cast<uintptr_t>(lv->conv2) | reinterpret_cast<uintptr_t>(lv->B)) % 16 == 0) &&
           (long long)lv->nb * lv->N < (1LL << 31) && (long long)lv->nb * ((lv->N + 63) / 64 + 80) < (1LL << 31) &&
           (long long)lv->h * lv->w * lv->conv2_channels < (1LL << 31) && tc_f2_width_ok(lv);
}

int build_plan_tc(const banet_level_t* lv, int num_sms, BuildPlan* plan)
{
    plan->KP = 128;
    if (lv->grid_w > 0) plan->tiles_per_pair = ((lv->grid_w + 7) / 8) * ((lv->grid_h + 7) / 8);
    else plan->tiles_per_pair = (lv->N + TC_TILE - 1) / TC_TILE;
    plan->total_tiles = (long long)lv->nb * plan->tiles_per_pair;
    long long grid = num_sms;
    if (grid > plan->total_tiles) grid = plan->total_tiles;
    if (grid < 1) grid = 1;
    plan->grid = (int)grid;
    const long long tiles_per_cta = (plan->total_tiles + grid - 1) / grid;
    plan->max_span = (int)((tiles_per_cta + plan->tiles_per_pair - 2) / plan->tiles_per_pair) + 1;
    SlotLayout L{lv->K, lv->C};
    plan->slot_floats = L.floats();
    plan->ws_bytes = align_up((size_t)plan->grid * plan->max_span * plan->slot_floats * sizeof(float), 256);
    return BANET_OK;
}

int lm_build_tc(const banet_level_t* lv, const BuildPlan& plan, int mode, const float* R, const float* T, const float* W,
                float* H, float* g, float* rbar_sum, float* nvalid, void* ws, cudaStream_t st)
{
    BANET_REQUIRE(tc_supported(lv), BANET_ERR_UNSUPPORTED,
                  "lm_build (tensor-core path) needs K in {32,64,128}, C in {64,128}, 16-B aligned tensors; got K=%d C=%d", lv->K, lv->C);
    const int kblk = lv->K / 32;
    if (kblk != 4 && mode == 1) mode = 2;          // K = 64 / 32: the single-pass mode is not instantiated
    CUtensorMap tm;
    int rc;
    const bool basis_bf16 = lv->basis_dtype == BANET_DTYPE_BF16;     // 32-column blocks either way: 128-B rows (fp32) or 64-B rows (bf16)
    if (lv->grid_w > 0) rc = make_tmap_basis_3d(&tm, lv->B, basis_bf16, (uint64_t)lv->nb * lv->grid_h, lv->grid_w, lv->K, 8, 8, 32);
    else rc = make_tmap_basis_2d(&tm, lv->B, basis_bf16, (uint64_t)lv->nb * lv->N, lv->K, TC_TILE, 32);
    if (rc) return rc;
    const bool fly = lv->conv2_channels == lv->C;
    BuildParams prm;
    prm.nb = lv->nb; prm.N = lv->N; prm.C = lv->C; prm.K = lv->K; prm.h = lv->h; prm.w = lv->w; prm.c2 = lv->conv2_channels;
    prm.conv1 = lv->conv1; prm.conv2 = lv->conv2; prm.intr = lv->intr; prm.p = lv->p; prm.D = lv->D; prm.B = lv->B;
    prm.R = R; prm.T = T; prm.W = W; prm.weight = lv->weight; prm.robust = lv->robust; prm.robust_scale = lv->robust_scale;
    prm.partials = reinterpret_cast<float*>(ws);
    prm.slot_floats = plan.slot_floats; prm.max_span = plan.max_span;
    prm.tiles_per_pair = plan.tiles_per_pair; prm.total_tiles = plan.total_tiles;
    prm.grid_w = lv->grid_w; prm.grid_h = lv->grid_h;
    prm.tiles_x = lv->grid_w > 0 ? (lv->grid_w + 7) / 8 : 0; prm.tiles_y = lv->grid_h > 0 ? (lv->grid_h + 7) / 8 : 0;
    prm.band_rows = 1; prm.l2_hints = 0; prm.tap_prefetch = 0; prm.kq_i = 0; prm.kq_j = 0;
    prm.hdd_transposed = 1;
    prm.trace = nullptr;
    const int nch = lv->C / 64;
    // dense grid: band walk + L2 policy (diagnostic knobs, off by default)
    int band = g_tuning.tc6_band_rows > 0 ? g_tuning.tc6_band_rows : kTc6DefaultBandRows;
    if (band > prm.tiles_y) band = prm.tiles_y;
    prm.band_rows = lv->grid_w > 0 && band > 1 ? band : 1;
    prm.l2_hints = g_tuning.tc6_l2_hints > 0 ? g_tuning.tc6_l2_hints - 1 : kTc6DefaultL2Hints;
    prm.tap_prefetch = g_tuning.tc6_tap_prefetch > 0 ? g_tuning.tc6_tap_prefetch - 1 : kTc6DefaultTapPrefetch;
    rc = lm_build_tc6_launch(mode, fly, nch, kblk, lv->feature_dtype == BANET_DTYPE_BF16, basis_bf16, tm, prm, plan.grid, st);
    if (rc) return rc;
    return launch_lm_reduce(prm, plan.grid, H, g, rbar_sum, nvalid, st);
}

}  // namespace banet
