// gsr_b200 — shared-memory vector accessors and two-lane fp32 (f32x2) helpers shared by the blend kernels.
#pragma once
#include "gsr_common.cuh"

namespace gsr {

__device__ __forceinline__ float4 lds128(uint32_t a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts128(uint32_t a, const float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ float2 lds64(uint32_t a) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a));
    return v;
}

// Two-lane fp32: the blend evaluates TWO queued splats per iteration, one per lane.  Hopper has no packed fp32
// instruction, so each lane is one IEEE round-to-nearest FFMA / FMUL / FADD; the _rn intrinsics keep nvcc from
// contracting a multiply and an add into one FMA, so every lane rounds exactly as the scalar formula it mirrors.
struct f32x2 {
    float lo, hi;
};
__device__ __forceinline__ f32x2 pk2(float lo, float hi) { return f32x2{lo, hi}; }
__device__ __forceinline__ void upk2(f32x2 v, float& lo, float& hi) {
    lo = v.lo;
    hi = v.hi;
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return f32x2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)}; }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return f32x2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return f32x2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
__device__ __forceinline__ float ex2_approx(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

}  // namespace gsr
