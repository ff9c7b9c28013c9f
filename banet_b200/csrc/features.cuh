// Element types of banet_level_t::feature_dtype and ::basis_dtype: float, or bf16 widened to fp32 exactly where it is read.
#pragma once
#include <cuda_bf16.h>
#include "common.cuh"

namespace banet {
typedef __nv_bfloat16 bf16;
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }          // element 2i of a packed pair
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }  // element 2i + 1
__device__ __forceinline__ float ldg_feat(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ldg_feat(const bf16* p) { return __uint_as_float((uint32_t)__ldg(reinterpret_cast<const unsigned short*>(p)) << 16); }
// 4 consecutive bf16 (8 B), streaming
__device__ __forceinline__ uint2 ld_stream_bf4(const bf16* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ float ld_stream_bf1(const bf16* p) {
    unsigned short r;
    asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(r) : "l"(p));
    return __uint_as_float((uint32_t)r << 16);
}
// one element of a read-once stream (the basis rows), widened
__device__ __forceinline__ float ld_stream_elem(const float* p) { return ld_stream_f1(p); }
__device__ __forceinline__ float ld_stream_elem(const bf16* p) { return ld_stream_bf1(p); }

}  // namespace banet
