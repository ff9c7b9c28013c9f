// sm_90a primitives used by the tensor-core build path: mbarrier, TMA (cp.async.bulk.tensor), the 128B swizzle and
// warp-level tf32 MMAs that read their fragments from the swizzled tiles.
// Inline PTX only; no CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace banet { namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}"
                 :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) { }
}

// wait with a hardware suspend-time hint: the warp is parked by the barrier unit (no issue slots burnt on polling) and woken on completion
__device__ __forceinline__ void mbar_wait_parked(uint64_t* bar, uint32_t parity) {
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
                 :: "r"(smem_u32(bar)), "r"(parity), "r"(0x989680) : "memory");
}
template <int NREG> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(NREG)); }
template <int NREG> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(NREG)); }

// generic-proxy writes (st.shared) -> visible to the async proxy (TMA)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" :: "l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load: box lands at `dst` (swizzled as the tensor map says), completes `bytes` on `bar`.
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// L2 eviction-priority policies (createpolicy) and the loads that carry one
__device__ __forceinline__ uint64_t l2_policy_evict_first()  { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint64_t l2_policy_evict_last()   { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint64_t l2_policy_evict_normal() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ void tma_load_2d_hint(void* dst, const CUtensorMap* m, int c0, int c1, uint64_t* bar, uint64_t pol) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(pol) : "memory");
}
__device__ __forceinline__ void tma_load_3d_hint(void* dst, const CUtensorMap* m, int c0, int c1, int c2, uint64_t* bar, uint64_t pol) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(pol) : "memory");
}
__device__ __forceinline__ float4 ld_stream_f4_hint(const float* p, uint64_t pol) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ float4 ldg4_hint(const float* p, uint64_t pol) {
    float4 r;
    asm("ld.global.nc.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p), "l"(pol));
    return r;
}

// L2 prefetch (no destination, no completion) of a contiguous range
__device__ __forceinline__ void prefetch_l2_bulk(const void* p, uint32_t bytes) {      // bytes % 16 == 0, p 16-B aligned
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(p), "r"(bytes) : "memory");
}

// ---------------------------------------------------------------- warp-level tf32 MMA on the swizzled tiles
// Both operands of the contraction D[i][n] = sum_px A[px][i] * R[px][n] lie pixel-major in shared memory (A as TMA lands the basis
// tile from HBM): they are MN-major.  Hopper's wgmma takes tf32 operands K-major only, so the fragments are read from the swizzled
// tiles by LDS and fed to mma.sync m16n8k8 (fp32 accumulate in registers).  Every fragment is truncated to tf32 explicitly (low 13
// bits cleared): the operand splitting of the precision modes (A_lo = b - trunc(b), R = rna(s*b) by +0x1000) relies on it.
__device__ __forceinline__ void mma_tf32_m16n8k8(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t lds_tf32(uint32_t saddr) {
    uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(saddr)); return v & 0xFFFFE000u;
}
// Byte offset, inside a tile of [64 px] x [32-column blocks of 128 B] (block stride 8192 B, 128B swizzle), of column `col` in
// pixel row 8*kk + r (r in 0..7; add kk * 1024).
__device__ __forceinline__ uint32_t frag_off(int col, int r) {
    return (uint32_t)((col >> 5) * 8192 + r * 128 + ((((col & 31) >> 2) ^ r) << 4) + (col & 3) * 4);
}
// A fragment (rows i0 .. i0+15 of A^T, pixels 8*kk .. 8*kk+7) from the tile at shared address `a`
__device__ __forceinline__ void load_a_frag(uint32_t (&f)[4], uint32_t a, int i0, int kk, int lane) {
    const int g = lane >> 2, t = lane & 3;
    a += kk * 1024;
    f[0] = lds_tf32(a + frag_off(i0 + g, t));     f[1] = lds_tf32(a + frag_off(i0 + g + 8, t));
    f[2] = lds_tf32(a + frag_off(i0 + g, t + 4)); f[3] = lds_tf32(a + frag_off(i0 + g + 8, t + 4));
}
// d += A^T[i0 .. i0+15][8 px] x R[8 px][n0 .. n0+7]
__device__ __forceinline__ void mma_step(float (&d)[4], const uint32_t (&af)[4], uint32_t r, int n0, int kk, int lane) {
    const int n = n0 + (lane >> 2), t = lane & 3;
    r += kk * 1024;
    mma_tf32_m16n8k8(d, af, lds_tf32(r + frag_off(n, t)), lds_tf32(r + frag_off(n, t + 4)));
}
// The same step for long sums: the tensor core forms the 8-pixel product from zero and it is added to d in round-to-nearest fp32
// (the build kernels' MMA role, mma_role.cuh: mma_add_rn, takes the same step on fragments it loads itself).
// The tensor core's own fp32 accumulation truncates (biased toward zero, see tests/test_gpu_tensorcore.py), which over the
// thousands of steps of a pair span would bias H_dd.
__device__ __forceinline__ void mma_step_rn(float (&d)[4], const uint32_t (&af)[4], uint32_t r, int n0, int kk, int lane) {
    float p[4] = {0.f, 0.f, 0.f, 0.f};
    mma_step(p, af, r, n0, kk, lane);
    d[0] += p[0]; d[1] += p[1]; d[2] += p[2]; d[3] += p[3];
}

// Byte offset of (row r, 16-byte chunk c in 0..7) inside one [rows][128 B] block in the 128B swizzle as TMA writes it
// (CU_TENSOR_MAP_SWIZZLE_128B, block base 1024-B aligned): the chunk index is XORed with (r & 7).
__device__ __forceinline__ uint32_t sw128_off(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }
// The same for one [rows][64 B] block in the 64B swizzle (CU_TENSOR_MAP_SWIZZLE_64B, block base 512-B aligned): address bits 4-5 are
// XORed with bits 7-8, so the 16-byte chunk index c in 0..3 is XORed with (r >> 1) & 3.  The bf16 basis tile: 32 columns per row.
__device__ __forceinline__ uint32_t sw64_off(int r, int c) { return (uint32_t)(r * 64 + ((c ^ ((r >> 1) & 3)) << 4)); }

__device__ __forceinline__ float tf32_rna(float x) {          // round to nearest tf32 (10-bit mantissa), ties away
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
// round-to-nearest (ties away) for an operand whose low 13 bits the tensor core ignores anyway: one integer add, no mask
__device__ __forceinline__ float tf32_rna_bits(float x) { return __uint_as_float(__float_as_uint(x) + 0x1000u); }
__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

}}  // namespace banet::tc
