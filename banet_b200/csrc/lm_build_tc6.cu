// lm_build_tc6.cu — tensor-core build kernel, generation 6: every phase has its own warpgroup, phases of different tiles overlap.
//
// Contract, slot layout and precision modes: see lm_build_tc_host.cu.  Roles (640 threads, 1 CTA / SM; register budgets by setmaxnreg,
// 48 / 112 / 72 / 136 = 61 440 registers, the CTA's allocation at 96 per thread):
//
//   warpgroup 0    4 geometry warps, 16 pixels each per tile, run ahead of everybody:                              (48 regs)
//                    b.W from the TMA-staged basis tile, warp / mask / tap offsets -> pixel records (ring of NREC)
//   warpgroups 1-2 8 gather warps, 8 pixels each per tile: records -> 13 tap loads -> blend / accumulate -> M, q, |d|^2  (112 regs)
//   warpgroup 3    4 algebra warps, 16 pixels each per tile:                                                        (72 regs)
//                    2x7 per-pixel algebra (H_cc / g_c partials in registers), R rows (A_lo, R_lo) into smem,
//                    refill of the freed basis stage by TMA (one elected thread)
//   warpgroup 4    4 MMA warps: D = A^T R of every tile by mma.sync tf32 (each 8-pixel step added round-to-nearest) into register
//                    accumulators that live for the whole pair span (lower block triangle of H_dd + the [v | t] columns, 80 floats per
//                    thread); one slot write per span (136 regs)
//   The accumulators take the registers the 5th-generation tensor core kept in tensor memory; half of the gather warps give them up.
//   mbarriers: fullB[NST] TMA landed | recs[NREC] geometry->gather | gath[NREC] gather->algebra | recfree[NREC] algebra->geometry |
//              rready R (A_lo, R_lo) of the tile written | rfree MMAs of the tile done (R, A_lo and the A stage reusable) |
//              rbdump/rbfree gather<->algebra hand-over of the |diff| sums at a pair change.
#include "common.cuh"
#include "features.cuh"
#include "lm_build.h"
#include "tc_utils.cuh"
#include "mma_role.cuh"
#include "tmap.h"
#include <stdlib.h>

namespace banet { namespace v6 {
using namespace tc;

constexpr int TILE = 64, W0 = 4, GW = 8, AW = 4, MW = 4;       // geometry | gather | algebra | MMA warps
constexpr int THREADS = (W0 + GW + AW + MW) * 32;               // 640
constexpr int STAGE_A = 4 * TILE * 128, STAGE_R = 5 * TILE * 128;
constexpr int REC = 16;

// BB: the basis is bf16.  Its stage holds the same 32-column blocks with 64-B rows (64B swizzle), half the bytes, and needs no A_lo
// tile: every bf16 value is exact in tf32, so the split-A pass multiplies zero.
template <int MODE, bool FLY, bool BB = false> struct Smem {
#ifndef BANET_TC6_NST1
#define BANET_TC6_NST1 4
#endif
#ifndef BANET_TC6_NST2
#define BANET_TC6_NST2 3
#endif
#ifndef BANET_TC6_NST3
#define BANET_TC6_NST3 2
#endif
#ifndef BANET_TC6_NREC
#define BANET_TC6_NREC 3
#endif
    // basis-tile stages (TMA ring) and pixel-record buffers per precision mode.  Deeper rings decouple the roles, but whatever smem the
    // CTA takes is lost to the L1, which holds the gather warps' tap loads in flight and catches the tap overlap of neighbouring pixels.
    static constexpr int NST = MODE == 1 ? BANET_TC6_NST1 : MODE == 2 ? BANET_TC6_NST2 : BANET_TC6_NST3;
    static constexpr int NREC = MODE == 3 ? 2 : BANET_TC6_NREC;
    static constexpr int STAGE = BB ? STAGE_A / 2 : STAGE_A;           // one basis-tile stage
    static constexpr int off_A = 0;
    static constexpr int off_R = NST * STAGE;
    static constexpr int off_Alo = off_R + STAGE_R;
    static constexpr int off_Rlo = off_Alo + (MODE >= 2 && !BB ? STAGE_A : 0);
    static constexpr int off_misc = off_Rlo + (MODE == 3 ? STAGE_R : 0);
    static constexpr int off_bar = off_misc;                           // 22 mbarriers
    static constexpr int off_tile = off_misc + 192;                    // [NREC][4] ints: pair index of the tile in record buffer s
    static constexpr int off_pose = off_tile + 64;                     // [W0][16] floats (private to each geometry warp)
    static constexpr int off_w = off_pose + W0 * 16 * 4;               // [W0][128] floats: W of the pair (private to each geometry warp)
    static constexpr int off_rec = off_w + W0 * 128 * 4;               // [NREC][TILE][REC] floats
    static constexpr int off_rbs = off_rec + NREC * TILE * REC * 4;    // [GW][128] floats: rbar hand-over gather -> algebra
    static constexpr int off_ccs = off_rbs + GW * 128 * 4;             // [AW][28] floats: H_cc / g_c / nvalid partials per algebra warp
    static constexpr int total = off_ccs + AW * 28 * 4;
    static constexpr int slack = 1024;                                 // stage bases 1024-B aligned (128B swizzle atoms)
    static constexpr int bytes = total + slack;
};

__device__ __forceinline__ long long gtime6() { long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
// debug timeline (BANET_TC_TRACE_PTR): CTA 1, gather warp 0 (role 0), algebra warp 0 (role 1) and geometry warp 0 (role 2), tiles 16..47, 12 stamps each
#ifdef BANET_TC6_TRACE_ON
#define TC6_TRACE(role, it, slot) do { if (prm.trace && blockIdx.x == 1 && lane == 0 && (it) >= 16 && (it) < 48) \
        prm.trace[(((role) * 32 + ((it) - 16)) * 12) + (slot)] = gtime6(); } while (0)
#else
#define TC6_TRACE(role, it, slot) do { } while (0)
#endif
template <int NT> __device__ __forceinline__ void team_bar() { asm volatile("bar.sync 2, %0;" :: "n"(NT) : "memory"); }
__device__ __forceinline__ int reflect_i(int i, int n) { i = i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); return i < 0 ? 0 : i; }
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float hsum16(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 8); v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}
struct TileCoord { int b, n0, cnt, tx0, ty0; };
__device__ __forceinline__ TileCoord tile_coord(const BuildParams& prm, long long tl) {
    TileCoord tc;
    const unsigned t = (unsigned)tl, tpp = (unsigned)prm.tiles_per_pair;
    tc.b = (int)(t / tpp);
    const int r = (int)(t - (unsigned)tc.b * tpp);
    if (prm.grid_w > 0) {
        int tyi, txi;
        if (prm.band_rows > 1) {        // bands of band_rows tile rows, column by column inside a band: vertically adjacent tiles follow each other
            const int bsz = prm.tiles_x * prm.band_rows, band = r / bsz, rem = r - band * bsz;
            const int rows = min(prm.band_rows, prm.tiles_y - band * prm.band_rows);
            txi = rem / rows; tyi = band * prm.band_rows + (rem - txi * rows);
        } else { tyi = r / prm.tiles_x; txi = r - tyi * prm.tiles_x; }
        tc.ty0 = tyi * 8; tc.tx0 = txi * 8; tc.n0 = 0; tc.cnt = TILE;
    }
    else { tc.n0 = r * TILE; tc.cnt = min(TILE, prm.N - tc.n0); tc.tx0 = tc.ty0 = 0; }
    return tc;
}

// ---- gather warps on bf16 features --------------------------------------------------------------------------------------------------
// Half-warp per pixel as for fp32; lane hl holds channels CPL*hl .. CPL*hl + CPL-1 (CPL = C/16), so each of the 13 taps is one 16-B
// (C = 128) or 8-B (C = 64) load.  At C = 64 this is the fp32 lane map and channel order (results bitwise equal to fp32 on the widened
// maps); at C = 128 a lane's 8 channels are contiguous instead of two groups of 4 64 apart, which reorders the per-pixel channel sums.
template <int CPL> struct BfTap;
template <> struct BfTap<8> {
    using T = uint4;
    static __device__ __forceinline__ T ld(const bf16* p, uint64_t pol) {
        T r; asm("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol)); return r; }
    static __device__ __forceinline__ T ld_stream(const bf16* p, uint64_t pol) {
        T r; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                          : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol)); return r; }
    static __device__ __forceinline__ float ch(const T& v, int i) {
        const uint32_t u = (i >> 1) == 0 ? v.x : (i >> 1) == 1 ? v.y : (i >> 1) == 2 ? v.z : v.w;
        return (i & 1) ? bf16_hi(u) : bf16_lo(u);
    }
};
template <> struct BfTap<4> {
    using T = uint2;
    static __device__ __forceinline__ T ld(const bf16* p, uint64_t pol) {
        T r; asm("ld.global.nc.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;" : "=r"(r.x), "=r"(r.y) : "l"(p), "l"(pol)); return r; }
    static __device__ __forceinline__ T ld_stream(const bf16* p, uint64_t pol) {
        T r; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;" : "=r"(r.x), "=r"(r.y) : "l"(p), "l"(pol)); return r; }
    static __device__ __forceinline__ float ch(const T& v, int i) {
        const uint32_t u = (i >> 1) == 0 ? v.x : v.y;
        return (i & 1) ? bf16_hi(u) : bf16_lo(u);
    }
};

template <int NCH, bool FLY, int NREC, bool ROBUST>
__device__ __forceinline__ void gather_bf16(const BuildParams& prm, const int* sTile, float* sRec, float* sRbs, uint64_t* recs, uint64_t* gath,
                                            uint64_t* rbdump, uint64_t* rbfree, int ntiles, int g, int lane)
{
    constexpr int C = 64 * NCH, CPL = C / 16, PXW = TILE / GW;
    using TB = BfTap<CPL>;
    const int hw = lane >> 4, hl = lane & 15;
    const int N = prm.N, h = prm.h, w = prm.w, c2 = prm.c2;
    float rb[CPL];
#pragma unroll
    for (int u = 0; u < CPL; ++u) rb[u] = 0.f;
    typename TB::T tb[13];
    int cur_b = -1, ndump = 0;
    const uint64_t pol_stream = prm.l2_hints >= 1 ? l2_policy_evict_first() : l2_policy_evict_normal();
    const uint64_t pol_tap = prm.l2_hints >= 2 ? l2_policy_evict_last() : l2_policy_evict_normal();

    auto dump_rb = [&]() {
        if (ndump > 0) mbar_wait_parked(rbfree, (ndump - 1) & 1);
#pragma unroll
        for (int u = 0; u < CPL; ++u) rb[u] += __shfl_xor_sync(0xffffffffu, rb[u], 16);
        if (hw == 0) {
#pragma unroll
            for (int j = 0; j < CPL / 4; ++j)
                *reinterpret_cast<float4*>(sRbs + g * 128 + CPL * hl + 4 * j) = make_float4(rb[4 * j], rb[4 * j + 1], rb[4 * j + 2], rb[4 * j + 3]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(rbdump);
#pragma unroll
        for (int u = 0; u < CPL; ++u) rb[u] = 0.f;
        ++ndump;
    };

    for (int j = 0; j < ntiles; ++j) {
        const int s = j % NREC;
        mbar_wait_parked(&recs[s], (j / NREC) & 1);
        const int b = sTile[s * 4];
        if (b != cur_b) { if (cur_b >= 0) dump_rb(); cur_b = b; }
        float* rec = sRec + (s * TILE + g * PXW) * REC;
        const bf16* c1b = static_cast<const bf16*>(prm.conv1) + (size_t)b * N * C + CPL * hl;
        const bf16* img = static_cast<const bf16*>(prm.conv2) + (size_t)b * h * w * c2 + CPL * hl;
#pragma unroll
        for (int u = 0; u < PXW / 2; ++u) {
            const int pl = 2 * u + hw;
            const float mask = rec[pl * REC + 4];
            float m11 = 0.f, m12 = 0.f, m22 = 0.f, q1 = 0.f, q2 = 0.f, ss = 0.f;
            if (mask != 0.f) {
                const uint4 o = *reinterpret_cast<const uint4*>(rec + pl * REC);
                const int n = __float_as_int(rec[pl * REC + 11]);
                auto ldt = [&](const bf16* q) { return TB::ld(q, pol_tap); };
                tb[0] = TB::ld_stream(c1b + (size_t)n * C, pol_stream);
                if constexpr (!FLY) {
                    const bf16* t00 = img + o.x; const bf16* t01 = img + o.y; const bf16* t10 = img + o.z; const bf16* t11 = img + o.w;
                    tb[1] = ldt(t00); tb[2] = ldt(t01); tb[3] = ldt(t10); tb[4] = ldt(t11);
                    tb[5] = ldt(t00 + C); tb[6] = ldt(t01 + C); tb[7] = ldt(t10 + C); tb[8] = ldt(t11 + C);
                    tb[9] = ldt(t00 + 2 * C); tb[10] = ldt(t01 + 2 * C); tb[11] = ldt(t10 + 2 * C); tb[12] = ldt(t11 + 2 * C);
                } else {
                    const uint2 cxy = *reinterpret_cast<const uint2*>(rec + pl * REC + 14);
                    const bf16* rm = img + o.x; const bf16* r0 = img + o.y; const bf16* r1 = img + o.z; const bf16* rp = img + o.w;
                    const uint32_t oM = (cxy.x & 0xffffu) * c2, o0 = (cxy.x >> 16) * c2, o1 = (cxy.y & 0xffffu) * c2, oP = (cxy.y >> 16) * c2;
                    tb[1] = ldt(r0 + oM); tb[2] = ldt(r0 + o0); tb[3] = ldt(r0 + o1); tb[4] = ldt(r0 + oP);      // aM0 a00 a10 aP0
                    tb[5] = ldt(r1 + oM); tb[6] = ldt(r1 + o0); tb[7] = ldt(r1 + o1); tb[8] = ldt(r1 + oP);      // aM1 a01 a11 aP1
                    tb[9] = ldt(rm + o0); tb[10] = ldt(rm + o1); tb[11] = ldt(rp + o0); tb[12] = ldt(rp + o1);   // a0m a1m a0p a1p
                }
                const float2 dxy = *reinterpret_cast<const float2*>(rec + pl * REC + 12);
                const float dx = dxy.x, dy = dxy.y;
                const float w00 = (1.f - dx) * (1.f - dy), w01 = dx * (1.f - dy), w10 = (1.f - dx) * dy, w11 = dx * dy;
                const float h00 = 0.5f * w00, h01 = 0.5f * w01, h10 = 0.5f * w10, h11 = 0.5f * w11;
#pragma unroll
                for (int i = 0; i < CPL; ++i) {
                    float t[13];
#pragma unroll
                    for (int k = 0; k < 13; ++k) t[k] = TB::ch(tb[k], i);
                    float f2, gx, gy;
                    if constexpr (!FLY) {
                        f2 = w00 * t[1] + w01 * t[2] + w10 * t[3] + w11 * t[4];
                        gx = w00 * t[5] + w01 * t[6] + w10 * t[7] + w11 * t[8];
                        gy = w00 * t[9] + w01 * t[10] + w10 * t[11] + w11 * t[12];
                    } else {
                        f2 = w00 * t[2] + w01 * t[3] + w10 * t[6] + w11 * t[7];
                        gx = h00 * (t[3] - t[1]) + h01 * (t[4] - t[2]) + h10 * (t[7] - t[5]) + h11 * (t[8] - t[6]);
                        gy = h00 * (t[6] - t[9]) + h10 * (t[11] - t[2]) + h01 * (t[7] - t[10]) + h11 * (t[12] - t[3]);
                    }
                    const float d = t[0] - f2;
                    m11 = fmaf(gx, gx, m11); m12 = fmaf(gx, gy, m12); m22 = fmaf(gy, gy, m22);
                    q1 = fmaf(gx, d, q1); q2 = fmaf(gy, d, q2);
                    if constexpr (ROBUST) ss = fmaf(d, d, ss);
                    rb[i] += fabsf(d);
                }
            }
            m11 = hsum16(m11); m12 = hsum16(m12); m22 = hsum16(m22); q1 = hsum16(q1); q2 = hsum16(q2);
            if constexpr (ROBUST) ss = hsum16(ss);
            if (hl == 0) {           // totals overwrite dx,dy / n of this pixel's record (as the fp32 gather does), times the point weight
                float wn = (prm.weight && mask != 0.f) ? __ldg(prm.weight + (size_t)b * N + __float_as_int(rec[pl * REC + 11])) : 1.f;
                if constexpr (ROBUST) wn *= robust_rho1(prm.robust, prm.robust_scale, ss);
                *reinterpret_cast<float4*>(rec + pl * REC + 12) = make_float4(m11 * wn, m12 * wn, m22 * wn, q1 * wn);
                rec[pl * REC + 11] = q2 * wn;
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&gath[s]);
    }
    if (cur_b >= 0) dump_rb();
}

// TF: feature element type (float or bf16).  bf16 keeps the half-warp per pixel; each tap is ONE load of the lane's C/16 channels
// (16 B of 8 channels at C = 128, 8 B of 4 at C = 64), widened channel by channel where it is used.
// TB: basis element type (float or bf16).  A bf16 tile is staged as it lies in HBM and widened in registers by each role that reads it:
// the b.W walk (same fp32 order), the R rows, the MMA's A fragments.  It is exact in tf32, so MODE 1 skips its in-place rounding and
// MODE 2 / 3 skip the split-A pass: results are bitwise those of the fp32 kernel on the widened basis.
// ROBUST: the gather warps also sum |d|^2 per pixel and weigh M, q by rho'(|d|^2) (banet_level_t::robust).  That is one more FFMA per
// channel and one more reduction per pixel on the warps suspected to pace the tile loop, so a non-robust level runs an instantiation
// without them: its code is that of a library without robust losses.
template <int NCH, bool FLY, int MODE, int KBLK = 4, typename TF = float, typename TB = float, bool ROBUST = false>
__global__ void __launch_bounds__(THREADS, 1)
lm_build_tc6_kernel(const __grid_constant__ CUtensorMap tmapB, const BuildParams prm)
{
    constexpr bool BB = sizeof(TB) == 2;
    using SM = Smem<MODE, FLY, BB>;
    constexpr int NST = SM::NST, NREC = SM::NREC;
    constexpr int BLK = BB ? 4096 : 8192;                            // bytes of one 32-column block of the basis tile
    // KBLK = K / 32 basis blocks actually present (K = 128, 64 or 32).  The smem geometry stays that of K = 128 (32-KB stages); blocks
    // >= KBLK are never loaded or read, and the [v | t] block of R follows the last one.
    constexpr int KR = 32 * KBLK, EXTB = KBLK;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    // align through the 32-bit shared address so that the compiler keeps every access in the shared state space (LDS/STS, not generic LD/ST)
    unsigned char* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + SM::off_bar);
    uint64_t* fullB = bars;            // [NST]  TMA landed
    uint64_t* rfree = bars + 4;        //        MMAs of the tile completed (count MW)
    uint64_t* rready = bars + 5;       //        R (A_lo, R_lo) of the tile written (count AW)
    uint64_t* recs = bars + 11;        // [NREC] records of the tile in buffer s written (count W0)
    uint64_t* gath = bars + 14;        // [NREC] M,q of the tile in buffer s written (count GW)
    uint64_t* recfree = bars + 17;     // [NREC] records of the tile in buffer s consumed by the algebra warps (count AW)
    uint64_t* rbdump = bars + 20;      //        gather warps parked their rbar partials (count GW)
    uint64_t* rbfree = bars + 21;      //        algebra warps consumed them (count AW)
    int* sTile = reinterpret_cast<int*>(base + SM::off_tile);
    float* sPose = reinterpret_cast<float*>(base + SM::off_pose);
    float* sW = reinterpret_cast<float*>(base + SM::off_w);
    float* sRec = reinterpret_cast<float*>(base + SM::off_rec);
    float* sRbs = reinterpret_cast<float*>(base + SM::off_rbs);
    float* sCcs = reinterpret_cast<float*>(base + SM::off_ccs);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int N = prm.N, h = prm.h, w = prm.w, c2 = prm.c2;
    const bool grid2d = prm.grid_w > 0;
    constexpr int C = 64 * NCH;
    const long long t_begin = part_begin(prm.total_tiles, gridDim.x, blockIdx.x);
    const long long t_end   = part_begin(prm.total_tiles, gridDim.x, blockIdx.x + 1);
    const int ntiles = (int)(t_end - t_begin);

    if (tid == 0) {
        for (int i = 0; i < NST; ++i) mbar_init(&fullB[i], 1);
        for (int i = 0; i < NREC; ++i) { mbar_init(&recs[i], W0); mbar_init(&gath[i], GW); mbar_init(&recfree[i], AW); }
        mbar_init(rfree, MW); mbar_init(rready, AW);
        mbar_init(rbdump, GW); mbar_init(rbfree, AW);
        fence_barrier_init();
        prefetch_tmap(&tmapB);
    }
    for (int i = tid; i < TILE * 8; i += THREADS) {       // pad chunks of R / R_lo's 5th block stay zero
        const int r = i >> 3, c = i & 7;
        *reinterpret_cast<float4*>(base + SM::off_R + EXTB * 8192 + sw128_off(r, c)) = make_float4(0.f, 0.f, 0.f, 0.f);
        if (MODE == 3) *reinterpret_cast<float4*>(base + SM::off_Rlo + EXTB * 8192 + sw128_off(r, c)) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();

    // lane -> (row r of the warp's 16, half hf of the 128 basis columns).  Every quarter-warp touches 8 distinct bank groups of the
    // swizzled tile: the b.W loop walks logical chunks in step (the swizzle spreads them; the W reads are broadcasts), the R-row loop
    // walks physical slots rotated by the row
    const int r16 = lane & 15, hf = lane >> 4;

    if (warp < W0) {
        // ===================================================================== geometry warps: b.W, warp, mask, tap offsets -> records
        setmaxnreg_dec<48>();
        const int gwi = warp, nlr = gwi * 16 + r16;
        float* myPose = sPose + gwi * 16;
        float* myW = sW + gwi * 128;
        int geom_b = -1;
        uint32_t dseed = 0;                                  // MODE 1: dither seed of the current pair
        TileCoord nxt = tile_coord(prm, t_begin);
        int nxt_r = (int)((unsigned)t_begin - (unsigned)nxt.b * (unsigned)prm.tiles_per_pair);
        for (int j = 0; j < ntiles; ++j) {
            const TileCoord tc = nxt;
            if (++nxt_r == prm.tiles_per_pair) { nxt_r = 0; ++nxt.b; nxt.tx0 = 0; nxt.ty0 = 0; nxt.n0 = 0; nxt.cnt = grid2d ? TILE : min(TILE, N); }
            else if (grid2d && prm.band_rows > 1) nxt = tile_coord(prm, t_begin + j + 1);
            else if (grid2d) { nxt.tx0 += 8; if (nxt.tx0 >= prm.tiles_x * 8) { nxt.tx0 = 0; nxt.ty0 += 8; } }
            else { nxt.n0 += TILE; nxt.cnt = min(TILE, N - nxt.n0); }
            const int b = tc.b;
            // No L2 bulk prefetch of the streaming inputs (conv1, p, D) ahead of the tile: issued two tiles ahead, it made the TF32X1 build
            // 10 % slower at 640x480 on H100, with bitwise the same outputs (DESIGN.md section 5).
            if (b != geom_b) {
                geom_b = b;
                __syncwarp();
                if (lane < 9) myPose[lane] = prm.R[b * 9 + lane];
                else if (lane < 12) myPose[lane] = prm.T[b * 3 + lane - 9];
                else if (lane < 16) myPose[lane] = prm.intr[b * 4 + lane - 12];
                if (KBLK == 4 || 4 * lane < KR)
                    *reinterpret_cast<float4*>(myW + 4 * lane) = __ldg(reinterpret_cast<const float4*>(prm.W + (size_t)b * KR + 4 * lane));
                if constexpr (MODE == 1)     // a pure function of the inputs that changes whenever the iterate changes (see the rounding below)
                    dseed = (__float_as_uint(__ldg(prm.W + (size_t)b * KR)) * 0x9E3779B1u) ^ (__float_as_uint(__ldg(prm.W + (size_t)b * KR + 1)) * 0x85EBCA77u)
                          ^ (__float_as_uint(__ldg(prm.W + (size_t)b * KR + 2)) * 0xC2B2AE3Du) ^ __float_as_uint(__ldg(prm.T + b * 3)) ^ (uint32_t)b;
                __syncwarp();
            }
            const int s = j % NST, sr = j % NREC;
            const unsigned char* As = base + SM::off_A + s * SM::STAGE;
            // global inputs of this lane's pixel first (their latency hides behind the waits and the dot product)
            float p0 = 0.f, p1 = 0.f, p2 = 0.f, D0 = 0.f;
            int n = 0; bool valid = false;
            if (grid2d) { const int gx = tc.tx0 + (nlr & 7), gy = tc.ty0 + (nlr >> 3); valid = gx < prm.grid_w && gy < prm.grid_h; n = gy * prm.grid_w + gx; }
            else { valid = nlr < tc.cnt; n = tc.n0 + nlr; }
            if (lane < 16 && valid) {
                const float* pp = prm.p + (size_t)b * 3 * N + n;
                p0 = __ldg(pp); p1 = __ldg(pp + N); p2 = __ldg(pp + 2 * (size_t)N);
                D0 = __ldg(prm.D + (size_t)b * N + n);
            }
            if (gwi == 0) TC6_TRACE(2, j, 0);
            mbar_wait_parked(&recfree[sr], ((j / NREC) & 1) ^ 1);
            mbar_wait_parked(&fullB[s], (j / NST) & 1);
            if (gwi == 0) TC6_TRACE(2, j, 1);
            float mydot;
            {
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                uint4 bq = make_uint4(0u, 0u, 0u, 0u);               // bf16: the 16-B chunk of columns 8(c/2) .. 8(c/2)+7, one LDS.128 per two steps
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int blk = 2 * hf + (i >> 3), c = i & 7;
                    if (KBLK != 4 && blk >= KBLK) continue;
                    float4 bv;
                    if constexpr (BB) {
                        if ((c & 1) == 0) bq = *reinterpret_cast<const uint4*>(As + blk * BLK + sw64_off(nlr, c >> 1));
                        const uint32_t u0 = (c & 1) ? bq.z : bq.x, u1 = (c & 1) ? bq.w : bq.y;
                        bv = make_float4(bf16_lo(u0), bf16_hi(u0), bf16_lo(u1), bf16_hi(u1));
                    } else {
                        bv = *reinterpret_cast<const float4*>(As + blk * 8192 + sw128_off(nlr, c));
                    }
                    const float4 w4 = *reinterpret_cast<const float4*>(myW + blk * 32 + c * 4);
                    acc.x = fmaf(bv.x, w4.x, acc.x); acc.y = fmaf(bv.y, w4.y, acc.y); acc.z = fmaf(bv.z, w4.z, acc.z); acc.w = fmaf(bv.w, w4.w, acc.w);
                    if constexpr (MODE == 1 && !BB) {
                        // single-pass mode: round the basis tile to tf32 IN PLACE.  The tensor core would truncate it (biased: relH 1e-5);
                        // round-to-nearest is unbiased per launch (relH < 1e-6) but is the SAME perturbation of the basis at every LM
                        // iteration, so its effect adds up coherently over a solve (W off by 1e-3 after 20 iterations).  Stochastic rounding
                        // with a dither hashed from (iterate, pixel, column) is unbiased AND changes with the iterate, like the rounding
                        // of R does; it is a pure function of the inputs, so results stay bit-reproducible.
                        uint32_t hsh = dseed ^ ((uint32_t)n * 0x9E3779B1u) ^ ((uint32_t)(blk * 8 + c) * 0x85EBCA77u);
                        hsh ^= hsh >> 16; hsh *= 0x7FEB352Du; hsh ^= hsh >> 15;
                        uint32_t hs2 = hsh * 0x846CA68Bu; hs2 ^= hs2 >> 16;
                        *reinterpret_cast<float4*>(const_cast<unsigned char*>(As) + blk * 8192 + sw128_off(nlr, c)) =
                            make_float4(__uint_as_float((__float_as_uint(bv.x) + (hsh & 0x1fffu)) & 0xFFFFE000u),
                                        __uint_as_float((__float_as_uint(bv.y) + ((hsh >> 13) & 0x1fffu)) & 0xFFFFE000u),
                                        __uint_as_float((__float_as_uint(bv.z) + (hs2 & 0x1fffu)) & 0xFFFFE000u),
                                        __uint_as_float((__float_as_uint(bv.w) + ((hs2 >> 13) & 0x1fffu)) & 0xFFFFE000u));
                    }
                }
                if constexpr (MODE == 1 && !BB) fence_proxy_async_smem();      // generic writes before the TMA refill of this stage
                mydot = (acc.x + acc.y) + (acc.z + acc.w);
                mydot += __shfl_xor_sync(0xffffffffu, mydot, 16);
            }
            if (gwi == 0) TC6_TRACE(2, j, 2);
            if (lane < 16) {                                 // thread per pixel (bundlenet.py:208-224, mask :231)
                const float* pose = myPose;
                float mask = 0.f, x = 0.f, y = 0.f, iZ = 0.f, rx = 0.f, ry = 0.f, rz = 0.f, dx = 0.f, dy = 0.f;
                int x0 = 0, y0 = 0;
                if (valid) {
                    const float Dt = D0 + mydot;
                    rx = pose[0] * p0 + pose[1] * p1 + pose[2] * p2;
                    ry = pose[3] * p0 + pose[4] * p1 + pose[5] * p2;
                    rz = pose[6] * p0 + pose[7] * p1 + pose[8] * p2;
                    const float X = rx * Dt + pose[9], Y = ry * Dt + pose[10], Z = rz * Dt + pose[11];
                    x = X / Z; y = Y / Z; iZ = 1.0f / Z;
                    const float u = pose[12] * x + pose[14], v = pose[13] * y + pose[15];
                    if ((u >= 0.f) && (u <= (float)(w - 1)) && (v >= 0.f) && (v <= (float)(h - 1)) && isfinite(iZ)) {
                        mask = 1.f;
                        const float fu = floorf(u), fv = floorf(v);
                        x0 = (int)fu; y0 = (int)fv; dx = u - fu; dy = v - fv;
                    }
                }
                uint32_t o[4], cx[2] = {0u, 0u};
                if constexpr (FLY) {                             // rows y0-1 .. y0+2 as float offsets, columns x0-1 .. x0+2 as packed pixel indices
                    o[0] = (uint32_t)(reflect_i(y0 - 1, h) * w * c2); o[1] = (uint32_t)(y0 * w * c2);
                    o[2] = (uint32_t)(reflect_i(y0 + 1, h) * w * c2); o[3] = (uint32_t)(reflect_i(y0 + 2, h) * w * c2);
                    cx[0] = (uint32_t)reflect_i(x0 - 1, w) | ((uint32_t)x0 << 16);
                    cx[1] = (uint32_t)reflect_i(x0 + 1, w) | ((uint32_t)reflect_i(x0 + 2, w) << 16);
                }
                if constexpr (!FLY) {
                    const int x1 = min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1);
                    o[0] = (uint32_t)((y0 * w + x0) * c2); o[1] = (uint32_t)((y0 * w + x1) * c2);
                    o[2] = (uint32_t)((y1 * w + x0) * c2); o[3] = (uint32_t)((y1 * w + x1) * c2);
                }
                if (prm.tap_prefetch && mask != 0.f) {
                    // pull this pixel's share of the tile's tap footprint into L2 one to two tiles before the gather warps load it: the gather is
                    // bound by the latency of its 13 dependent-free loads, not by their count.  Interior pixels fetch their (x0, y0) texel only;
                    // the tile's border pixels add the halo, so that under a near-unit warp every texel is requested about once.
                    const TF* imgp = static_cast<const TF*>(prm.conv2) + (size_t)b * h * w * c2;
                    const int px = nlr & 7, py = nlr >> 3;
                    const bool edge_x = !grid2d || px == 7, edge_y = !grid2d || py == 7 || prm.tap_prefetch == 2;
                    if constexpr (!FLY) {
                        const uint32_t by = (uint32_t)c2 * (uint32_t)sizeof(TF);
                        prefetch_l2_bulk(imgp + o[0], by);
                        if (edge_x && o[1] != o[0]) prefetch_l2_bulk(imgp + o[1], by);
                        if (edge_y && o[2] != o[0]) {
                            prefetch_l2_bulk(imgp + o[2], by);
                            if (edge_x && o[3] != o[2]) prefetch_l2_bulk(imgp + o[3], by);
                        }
                    } else {
                        const bool first_x = !grid2d || px == 0, first_y = !grid2d || py == 0;
                        const int xs = max(x0 - (first_x ? 1 : 0), 0), xe = min(x0 + (edge_x ? 2 : 0), w - 1);
                        const uint32_t by = (uint32_t)(xe - xs + 1) * (uint32_t)c2 * (uint32_t)sizeof(TF);
                        prefetch_l2_bulk(imgp + ((size_t)y0 * w + xs) * c2, by);
                        if (first_y && y0 > 0) prefetch_l2_bulk(imgp + ((size_t)(y0 - 1) * w + xs) * c2, by);
                        if (edge_y) {
                            if (y0 + 1 < h) prefetch_l2_bulk(imgp + ((size_t)(y0 + 1) * w + xs) * c2, by);
                            if (y0 + 2 < h) prefetch_l2_bulk(imgp + ((size_t)(y0 + 2) * w + xs) * c2, by);
                        }
                    }
                }
                float* rec = sRec + (sr * TILE + nlr) * REC;
                *reinterpret_cast<uint4*>(rec) = make_uint4(o[0], o[1], o[2], o[3]);
                *reinterpret_cast<float4*>(rec + 4) = make_float4(mask, x, y, iZ);
                *reinterpret_cast<float4*>(rec + 8) = make_float4(rx, ry, rz, __int_as_float(valid ? n : 0));
                *reinterpret_cast<float4*>(rec + 12) = make_float4(dx, dy, __uint_as_float(cx[0]), __uint_as_float(cx[1]));
            }
            if (gwi == 0 && lane == 0) sTile[sr * 4] = b;
            __syncwarp();
            if (gwi == 0) TC6_TRACE(2, j, 3);
            if (lane == 0) mbar_arrive(&recs[sr]);
        }
    } else if (warp < W0 + GW) {
        // ===================================================================== gather warps: records -> taps -> M, q
        setmaxnreg_inc<112>();
        if constexpr (sizeof(TF) == 2) { gather_bf16<NCH, FLY, NREC, ROBUST>(prm, sTile, sRec, sRbs, recs, gath, rbdump, rbfree, ntiles, warp - W0, lane); return; }
        const int g = warp - W0, hw = lane >> 4, hl = lane & 15;
        constexpr int PXW = TILE / GW;                       // 8 pixels per warp and tile
        constexpr int NUNIT = (PXW / 2) * NCH;
        float rb[NCH * 4];
#pragma unroll
        for (int u = 0; u < NCH * 4; ++u) rb[u] = 0.f;
        float4 tb[13];
        float m11 = 0.f, m12 = 0.f, m22 = 0.f, q1 = 0.f, q2 = 0.f, ss = 0.f;
        int cur_b = -1, ndump = 0;
        // L2 policy: conv1 is read exactly once (evict-first), the taps are what neighbouring tiles re-read
        const uint64_t pol_stream = prm.l2_hints >= 1 ? l2_policy_evict_first() : l2_policy_evict_normal();
        const uint64_t pol_tap = prm.l2_hints >= 2 ? l2_policy_evict_last() : l2_policy_evict_normal();

        auto dump_rb = [&]() {
            if (ndump > 0) mbar_wait_parked(rbfree, (ndump - 1) & 1);       // the algebra warps consumed the previous hand-over
#pragma unroll
            for (int u = 0; u < NCH * 4; ++u) rb[u] += __shfl_xor_sync(0xffffffffu, rb[u], 16);
            if (hw == 0) {
#pragma unroll
                for (int j = 0; j < NCH; ++j)
                    *reinterpret_cast<float4*>(sRbs + g * 128 + 64 * j + 4 * hl) = make_float4(rb[4 * j], rb[4 * j + 1], rb[4 * j + 2], rb[4 * j + 3]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(rbdump);
#pragma unroll
            for (int u = 0; u < NCH * 4; ++u) rb[u] = 0.f;
            ++ndump;
        };

        for (int j = 0; j < ntiles; ++j) {
            const int s = j % NREC;
            if (g == 0) TC6_TRACE(0, j, 0);
            mbar_wait_parked(&recs[s], (j / NREC) & 1);
            if (g == 0) TC6_TRACE(0, j, 1);
            const int b = sTile[s * 4];
            if (b != cur_b) { if (cur_b >= 0) dump_rb(); cur_b = b; }
            float* rec = sRec + (s * TILE + g * PXW) * REC;
            const float* c1b = static_cast<const float*>(prm.conv1) + (size_t)b * N * C + 4 * hl;
            const float* imgb = static_cast<const float*>(prm.conv2) + (size_t)b * h * w * c2 + 4 * hl;
#pragma unroll
            for (int u = 0; u < NUNIT; ++u) {
                const int pl = 2 * (u / NCH) + hw, co = 64 * (u % NCH), jc = u % NCH;
                const float mask = rec[pl * REC + 4];
                if (mask != 0.f) {
                    const uint4 o = *reinterpret_cast<const uint4*>(rec + pl * REC);
                    const int n = __float_as_int(rec[pl * REC + 11]);
                    const float* img = imgb + co;
                    auto ldt = [&](const float* q) { return ldg4_hint(q, pol_tap); };
                    tb[0] = ld_stream_f4_hint(c1b + (size_t)n * C + co, pol_stream);
                    if constexpr (!FLY) {
                        const float* t00 = img + o.x; const float* t01 = img + o.y; const float* t10 = img + o.z; const float* t11 = img + o.w;
                        tb[1] = ldt(t00); tb[2] = ldt(t01); tb[3] = ldt(t10); tb[4] = ldt(t11);
                        tb[5] = ldt(t00 + C); tb[6] = ldt(t01 + C); tb[7] = ldt(t10 + C); tb[8] = ldt(t11 + C);
                        tb[9] = ldt(t00 + 2 * C); tb[10] = ldt(t01 + 2 * C); tb[11] = ldt(t10 + 2 * C); tb[12] = ldt(t11 + 2 * C);
                    } else {
                        const uint2 cxy = *reinterpret_cast<const uint2*>(rec + pl * REC + 14);
                        const float* rm = img + o.x; const float* r0 = img + o.y; const float* r1 = img + o.z; const float* rp = img + o.w;
                        const uint32_t oM = (cxy.x & 0xffffu) * c2, o0 = (cxy.x >> 16) * c2, o1 = (cxy.y & 0xffffu) * c2, oP = (cxy.y >> 16) * c2;
                        tb[1] = ldt(r0 + oM); tb[2] = ldt(r0 + o0); tb[3] = ldt(r0 + o1); tb[4] = ldt(r0 + oP);      // aM0 a00 a10 aP0
                        tb[5] = ldt(r1 + oM); tb[6] = ldt(r1 + o0); tb[7] = ldt(r1 + o1); tb[8] = ldt(r1 + oP);      // aM1 a01 a11 aP1
                        tb[9] = ldt(rm + o0); tb[10] = ldt(rm + o1); tb[11] = ldt(rp + o0); tb[12] = ldt(rp + o1);   // a0m a1m a0p a1p
                    }
                }
                if (jc == 0) { m11 = m12 = m22 = q1 = q2 = ss = 0.f; }
                if (mask != 0.f) {
                    const float2 dxy = *reinterpret_cast<const float2*>(rec + pl * REC + 12);
                    const float dx = dxy.x, dy = dxy.y;
                    const float w00 = (1.f - dx) * (1.f - dy), w01 = dx * (1.f - dy), w10 = (1.f - dx) * dy, w11 = dx * dy;
                    const float4* t = tb;
                    if constexpr (!FLY) {
#define BANET_CH(F, CI)                                                                                              \
                        {                                                                                            \
                            const float f2 = w00 * t[1].F + w01 * t[2].F + w10 * t[3].F + w11 * t[4].F;              \
                            const float gx = w00 * t[5].F + w01 * t[6].F + w10 * t[7].F + w11 * t[8].F;              \
                            const float gy = w00 * t[9].F + w01 * t[10].F + w10 * t[11].F + w11 * t[12].F;           \
                            const float d = t[0].F - f2;                                                             \
                            m11 = fmaf(gx, gx, m11); m12 = fmaf(gx, gy, m12); m22 = fmaf(gy, gy, m22);               \
                            q1 = fmaf(gx, d, q1); q2 = fmaf(gy, d, q2);                                              \
                            if constexpr (ROBUST) ss = fmaf(d, d, ss);                                               \
                            rb[4 * jc + CI] += fabsf(d);                                                             \
                        }
                        BANET_CH(x, 0) BANET_CH(y, 1) BANET_CH(z, 2) BANET_CH(w, 3)
#undef BANET_CH
                    } else {
                        const float h00 = 0.5f * w00, h01 = 0.5f * w01, h10 = 0.5f * w10, h11 = 0.5f * w11;
#define BANET_CH(F, CI)                                                                                              \
                        {                                                                                            \
                            const float f2 = w00 * t[2].F + w01 * t[3].F + w10 * t[6].F + w11 * t[7].F;              \
                            const float gx = h00 * (t[3].F - t[1].F) + h01 * (t[4].F - t[2].F)                       \
                                           + h10 * (t[7].F - t[5].F) + h11 * (t[8].F - t[6].F);                      \
                            const float gy = h00 * (t[6].F - t[9].F) + h10 * (t[11].F - t[2].F)                      \
                                           + h01 * (t[7].F - t[10].F) + h11 * (t[12].F - t[3].F);                    \
                            const float d = t[0].F - f2;                                                             \
                            m11 = fmaf(gx, gx, m11); m12 = fmaf(gx, gy, m12); m22 = fmaf(gy, gy, m22);               \
                            q1 = fmaf(gx, d, q1); q2 = fmaf(gy, d, q2);                                              \
                            if constexpr (ROBUST) ss = fmaf(d, d, ss);                                               \
                            rb[4 * jc + CI] += fabsf(d);                                                             \
                        }
                        BANET_CH(x, 0) BANET_CH(y, 1) BANET_CH(z, 2) BANET_CH(w, 3)
#undef BANET_CH
                    }
                }
                if (jc == NCH - 1) {
                    m11 = hsum16(m11); m12 = hsum16(m12); m22 = hsum16(m22); q1 = hsum16(q1); q2 = hsum16(q2);
                    if constexpr (ROBUST) ss = hsum16(ss);
                    if (hl == 0) {           // totals overwrite dx,dy / n of this pixel's record (no longer needed; the tap offsets stay for the prefetcher)
                        // point weight times the robust loss's rho'(s) (M and q, i.e. every block of H and g; sum |d| stays unweighted):
                        // x * 1.0f is exact
                        float wn = (prm.weight && mask != 0.f) ? __ldg(prm.weight + (size_t)b * N + __float_as_int(rec[pl * REC + 11])) : 1.f;
                        if constexpr (ROBUST) wn *= robust_rho1(prm.robust, prm.robust_scale, ss);
                        *reinterpret_cast<float4*>(rec + pl * REC + 12) = make_float4(m11 * wn, m12 * wn, m22 * wn, q1 * wn);
                        rec[pl * REC + 11] = q2 * wn;
                    }
                }
            }
            __syncwarp();
            if (g == 0) TC6_TRACE(0, j, 2);
            if (lane == 0) mbar_arrive(&gath[s]);
        }
        if (cur_b >= 0) dump_rb();
    } else if (warp < W0 + GW + AW) {
        // ===================================================================== algebra warps: 2x7 algebra, R rows, TMA issue
        setmaxnreg_dec<72>();
        const int awi = warp - (W0 + GW);                    // 0..3: pixels / rows 16*awi .. 16*awi+15
        const int atid = tid - (W0 + GW) * 32;
        const int nlr = awi * 16 + r16;
        const SlotLayout L{KR, C};
        unsigned char* Rs = base + SM::off_R;
        float cc[28];
#pragma unroll
        for (int q = 0; q < 28; ++q) cc[q] = 0.f;
        int scale_b = -1, sspan = -1;
        float fx = 0.f, fy = 0.f;
        int rr = (ntiles > 0) ? (int)((unsigned)t_begin % (unsigned)prm.tiles_per_pair) : 0;
        const uint64_t pol_basis = prm.l2_hints >= 1 ? l2_policy_evict_first() : l2_policy_evict_normal();     // the basis is read exactly once
        auto issue_tma = [&](int t) {                        // basis tile t -> stage t % NST (elected thread)
            const int st = t % NST;
            const TileCoord tc = tile_coord(prm, t_begin + t);
            mbar_arrive_expect_tx(&fullB[st], KBLK * BLK);
            unsigned char* dst = base + SM::off_A + st * SM::STAGE;
            if (grid2d) {
#pragma unroll
                for (int blk = 0; blk < KBLK; ++blk) tma_load_3d_hint(dst + blk * BLK, &tmapB, blk * 32, tc.tx0, tc.b * prm.grid_h + tc.ty0, &fullB[st], pol_basis);
            } else {
                const int row = tc.b * N + tc.n0;
#pragma unroll
                for (int blk = 0; blk < KBLK; ++blk) tma_load_2d_hint(dst + blk * BLK, &tmapB, blk * 32, row, &fullB[st], pol_basis);
            }
        };
        auto flush = [&](int sp) {               // H_cc / g_c / nvalid and rbar of the span (the MMA warps write H_dd and the [v | t] columns)
            float* slot = prm.partials + ((size_t)blockIdx.x * prm.max_span + sp) * prm.slot_floats;
            // H_cc / g_c / nvalid: 16 pixel-lanes -> warp total (fixed shuffle tree) -> 4 warp partials summed in fixed order
#pragma unroll
            for (int q = 0; q < 28; ++q) {
                float v = cc[q];
                v += __shfl_xor_sync(0xffffffffu, v, 8); v += __shfl_xor_sync(0xffffffffu, v, 4);
                v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 1);
                if (lane == 0) sCcs[awi * 28 + q] = v;
                cc[q] = 0.f;
            }
            mbar_wait_parked(rbdump, sp & 1);                // the gather warps parked their |diff| sums for this pair
            team_bar<AW * 32>();
            if (atid < C) {
                float sum = 0.f;
#pragma unroll
                for (int wq = 0; wq < GW; ++wq) sum += sRbs[wq * 128 + atid];
                slot[L.off_rbar() + atid] = sum;
            }
            if (atid < 28) slot[L.off_cc() + atid] = (sCcs[atid] + sCcs[28 + atid]) + (sCcs[56 + atid] + sCcs[84 + atid]);
            team_bar<AW * 32>();
            if (lane == 0) mbar_arrive(rbfree);
        };

        if (awi == 0 && lane == 0)
            for (int t = 0; t < NST && t < ntiles; ++t) issue_tma(t);      // every stage starts free

        for (int j = 0; j < ntiles; ++j) {
            const int s = j % NST, sr = j % NREC;
            const bool last_of_pair = (++rr == prm.tiles_per_pair) || (j == ntiles - 1);
            if (rr == prm.tiles_per_pair) rr = 0;
            const unsigned char* As = base + SM::off_A + s * SM::STAGE;
            if (awi == 0) TC6_TRACE(1, j, 0);
            mbar_wait_parked(&gath[sr], (j / NREC) & 1);
            if (awi == 0) TC6_TRACE(1, j, 1);
            const int b = sTile[sr * 4];
            if (b != scale_b) { scale_b = b; ++sspan; fx = __ldg(prm.intr + b * 4); fy = __ldg(prm.intr + b * 4 + 1); }
            float ext[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (lane < 16) {                                 // thread per pixel (bundlenet.py:49-74)
                const float* rec = sRec + (sr * TILE + nlr) * REC;
                const float4 ra = *reinterpret_cast<const float4*>(rec + 12), rbq = *reinterpret_cast<const float4*>(rec + 4),
                             rc = *reinterpret_cast<const float4*>(rec + 8);
                if (rbq.x != 0.f) {
                    const float m11 = ra.x, m12 = ra.y, m22 = ra.z, q1 = ra.w, q2 = rc.w, x = rbq.y, y = rbq.z, iZ = rbq.w;
                    const float rx = rc.x, ry = rc.y, rz = rc.z;
                    const float a0[6] = {-fx * (x * y), -fx * (-1.f - x * x), -fx * y, -fx * (-iZ), 0.f, -fx * (x * iZ)};
                    const float a1[6] = {-fy * (1.f + y * y), -fy * (-(x * y)), -fy * (-x), 0.f, -fy * (-iZ), -fy * (y * iZ)};
                    float ux[6], uy[6];
#pragma unroll
                    for (int i = 0; i < 6; ++i) { ux[i] = m11 * a0[i] + m12 * a1[i]; uy[i] = m12 * a0[i] + m22 * a1[i]; }
                    int q = 0;
#pragma unroll
                    for (int i = 0; i < 6; ++i)
#pragma unroll
                        for (int jj = i; jj < 6; ++jj) { cc[q] += a0[i] * ux[jj] + a1[i] * uy[jj]; ++q; }
#pragma unroll
                    for (int i = 0; i < 6; ++i) cc[21 + i] += a0[i] * q1 + a1[i] * q2;
                    cc[27] += 1.f;
                    const float jd0 = fx * ((rx - rz * x) * iZ), jd1 = fy * ((ry - rz * y) * iZ);
                    const float u0 = m11 * jd0 + m12 * jd1, u1 = m12 * jd0 + m22 * jd1;
#pragma unroll
                    for (int i = 0; i < 6; ++i) ext[i] = a0[i] * u0 + a1[i] * u1;
                    ext[6] = jd0 * q1 + jd1 * q2;
                    ext[7] = jd0 * u0 + jd1 * u1;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&recfree[sr]);        // the record buffer may be refilled (everything needed is in registers)
            const float sn = __shfl_sync(0xffffffffu, ext[7], r16);   // s_n of this lane's row
            if (awi == 0) TC6_TRACE(1, j, 2);
            mbar_wait_parked(&fullB[s], (j / NST) & 1);      // long complete; orders the TMA writes before the reads below
            if (j > 0) {
                mbar_wait_parked(rfree, (j - 1) & 1);        // MMAs of tile j-1 done: R / A_lo / R_lo and stage (j-1) % NST are free
                if (awi == 0 && lane == 0 && j - 1 + NST < ntiles) issue_tma(j - 1 + NST);
            }
            if (awi == 0) TC6_TRACE(1, j, 3);
            if (lane < 16) {                                 // R columns 128..134 = [v(6) | t], column 135 stays zero
                const float4 e0 = make_float4(tf32_rna(ext[0]), tf32_rna(ext[1]), tf32_rna(ext[2]), tf32_rna(ext[3]));
                const float4 e1 = make_float4(tf32_rna(ext[4]), tf32_rna(ext[5]), tf32_rna(ext[6]), 0.f);
                *reinterpret_cast<float4*>(Rs + EXTB * 8192 + sw128_off(nlr, 0)) = e0;
                *reinterpret_cast<float4*>(Rs + EXTB * 8192 + sw128_off(nlr, 1)) = e1;
                if constexpr (MODE == 3) {
                    *reinterpret_cast<float4*>(base + SM::off_Rlo + EXTB * 8192 + sw128_off(nlr, 0)) = make_float4(ext[0] - e0.x, ext[1] - e0.y, ext[2] - e0.z, ext[3] - e0.w);
                    *reinterpret_cast<float4*>(base + SM::off_Rlo + EXTB * 8192 + sw128_off(nlr, 1)) = make_float4(ext[4] - e1.x, ext[5] - e1.y, ext[6] - e1.z, 0.f);
                }
            }
            // R rows (and the split parts): elementwise on the lane's half row, so walk the PHYSICAL 16-B slots (rotated by the row: every
            // quarter-warp touches 8 distinct bank groups) and skip the swizzle arithmetic
            if constexpr (BB) {
                // bf16 tile: walk the lane's 16-B chunks (8 columns each, logical chunk m of block blk, every quarter-warp on 8 distinct bank
                // groups), widen, and write the two fp32 chunks 2m, 2m+1 of the R row
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int blk = 2 * hf + (i >> 2), m = i & 3;
                    if (KBLK != 4 && blk >= KBLK) continue;
                    const uint4 q = *reinterpret_cast<const uint4*>(As + blk * BLK + sw64_off(nlr, m));
                    const float bw[8] = {bf16_lo(q.x), bf16_hi(q.x), bf16_lo(q.y), bf16_hi(q.y), bf16_lo(q.z), bf16_hi(q.z), bf16_lo(q.w), bf16_hi(q.w)};
#pragma unroll
                    for (int hc = 0; hc < 2; ++hc) {
                        const uint32_t off = blk * 8192 + sw128_off(nlr, 2 * m + hc);
                        const float4 pv = make_float4(sn * bw[4 * hc], sn * bw[4 * hc + 1], sn * bw[4 * hc + 2], sn * bw[4 * hc + 3]);
                        float4 hv;
                        if constexpr (MODE == 3) hv = make_float4(tf32_rna(pv.x), tf32_rna(pv.y), tf32_rna(pv.z), tf32_rna(pv.w));
                        else hv = make_float4(tf32_rna_bits(pv.x), tf32_rna_bits(pv.y), tf32_rna_bits(pv.z), tf32_rna_bits(pv.w));
                        *reinterpret_cast<float4*>(Rs + off) = hv;
                        if constexpr (MODE == 3)
                            *reinterpret_cast<float4*>(base + SM::off_Rlo + off) = make_float4(pv.x - hv.x, pv.y - hv.y, pv.z - hv.z, pv.w - hv.w);
                    }
                }
            } else {
            const uint32_t rowoff = hf * 16384 + nlr * 128;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                if (KBLK != 4 && 2 * hf + (i >> 3) >= KBLK) continue;
                const uint32_t off = rowoff + (i >> 3) * 8192 + (((i & 7) + r16) & 7) * 16;
                const float4 bv = *reinterpret_cast<const float4*>(As + off);
                const float4 pv = make_float4(sn * bv.x, sn * bv.y, sn * bv.z, sn * bv.w);
                float4 hv;
                if constexpr (MODE == 3) hv = make_float4(tf32_rna(pv.x), tf32_rna(pv.y), tf32_rna(pv.z), tf32_rna(pv.w));
                else hv = make_float4(tf32_rna_bits(pv.x), tf32_rna_bits(pv.y), tf32_rna_bits(pv.z), tf32_rna_bits(pv.w));   // MMA drops the low 13 bits
                *reinterpret_cast<float4*>(Rs + off) = hv;
                if constexpr (MODE >= 2)
                    *reinterpret_cast<float4*>(base + SM::off_Alo + off) = make_float4(bv.x - tf32_trunc(bv.x), bv.y - tf32_trunc(bv.y), bv.z - tf32_trunc(bv.z), bv.w - tf32_trunc(bv.w));
                if constexpr (MODE == 3)
                    *reinterpret_cast<float4*>(base + SM::off_Rlo + off) = make_float4(pv.x - hv.x, pv.y - hv.y, pv.z - hv.z, pv.w - hv.w);
            }
            }
            if (awi == 0) TC6_TRACE(1, j, 4);
            __syncwarp();
            if (lane == 0) mbar_arrive(rready);
            if (awi == 0) TC6_TRACE(1, j, 5);
            if (last_of_pair) flush(sspan);
        }
    } else {
        // ===================================================================== MMA warps: D = A^T R per tile, accumulated over the pair span
        setmaxnreg_inc<136>();
        mma_role<SM, SM::STAGE, MODE, KR, BB>(prm, base, fullB, rready, rfree, t_begin, ntiles, warp - (W0 + GW + AW), lane);
    }
}

template <int NCH, bool FLY, int MODE, int KBLK, typename TF, typename TB>
static int launch6(const CUtensorMap& tm, const BuildParams& prm, int grid, cudaStream_t st)
{
    auto kern = prm.robust ? lm_build_tc6_kernel<NCH, FLY, MODE, KBLK, TF, TB, true> : lm_build_tc6_kernel<NCH, FLY, MODE, KBLK, TF, TB, false>;
    const int smem = Smem<MODE, FLY, sizeof(TB) == 2>::bytes;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { set_error("lm_build_tc6: smem attr (%d B): %s", smem, cudaGetErrorString(e)); return BANET_ERR_CUDA; }
    kern<<<grid, THREADS, smem, st>>>(tm, prm);
    BANET_CUDA_LAUNCH_CHECK("lm_build_tc6_kernel launch");
    return BANET_OK;
}
template <int NCH, bool FLY, typename TF, typename TB>
static int launch6_mode(int mode, int kblk, const CUtensorMap& tm, const BuildParams& prm, int grid, cudaStream_t st)
{
    if (kblk != 4) {             // K = 64 / 32 (opt-in, BANET_TC_SMALLK=1): instantiated for the two-pass and the fp32-grade mode only
        if (kblk == 2) return mode == 3 ? launch6<NCH, FLY, 3, 2, TF, TB>(tm, prm, grid, st) : launch6<NCH, FLY, 2, 2, TF, TB>(tm, prm, grid, st);
        return mode == 3 ? launch6<NCH, FLY, 3, 1, TF, TB>(tm, prm, grid, st) : launch6<NCH, FLY, 2, 1, TF, TB>(tm, prm, grid, st);
    }
    if (mode == 1) return launch6<NCH, FLY, 1, 4, TF, TB>(tm, prm, grid, st);
    if (mode == 2) return launch6<NCH, FLY, 2, 4, TF, TB>(tm, prm, grid, st);
    return launch6<NCH, FLY, 3, 4, TF, TB>(tm, prm, grid, st);
}
template <typename TF, typename TB>
static int launch6_type(int mode, bool fly, int nch, int kblk, const CUtensorMap& tm, const BuildParams& prm, int grid, cudaStream_t st)
{
    if (nch == 2) return fly ? launch6_mode<2, true, TF, TB>(mode, kblk, tm, prm, grid, st) : launch6_mode<2, false, TF, TB>(mode, kblk, tm, prm, grid, st);
    return fly ? launch6_mode<1, true, TF, TB>(mode, kblk, tm, prm, grid, st) : launch6_mode<1, false, TF, TB>(mode, kblk, tm, prm, grid, st);
}

}  // namespace v6

int lm_build_tc6_launch(int mode, bool fly, int nch, int kblk, bool is_bf16, bool basis_bf16, const CUtensorMap& tm, const BuildParams& prm, int grid,
                        cudaStream_t st)
{
    if (basis_bf16)
        return is_bf16 ? v6::launch6_type<bf16, bf16>(mode, fly, nch, kblk, tm, prm, grid, st) : v6::launch6_type<float, bf16>(mode, fly, nch, kblk, tm, prm, grid, st);
    return is_bf16 ? v6::launch6_type<bf16, float>(mode, fly, nch, kblk, tm, prm, grid, st) : v6::launch6_type<float, float>(mode, fly, nch, kblk, tm, prm, grid, st);
}

}  // namespace banet
