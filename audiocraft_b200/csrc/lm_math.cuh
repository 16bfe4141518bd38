// Element arithmetic shared by the LM decode step (lm.cu) and the LM full-sequence forward (lm_forward.cu), so that both
// paths round and reduce the same way.
#pragma once
#include "common.cuh"

__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float half_round(float v) { return __half2float(__float2half_rn(v)); }
// v rounded to the nearest TF32 value (10-bit mantissa).  The TF32 wgmma drops an fp32 operand's low 13 bits (truncation);
// operands rounded first carry half that error.
__device__ __forceinline__ float tf32_round(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
}
__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f)); }

// Block reductions: every thread returns the full result; red needs >= 32 floats and may be reused right after
// the call returns only behind another barrier (callers alternate two scratch arrays).
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = lane < nw ? red[lane] : 0.f;
    return warp_sum(t);
}
