// Shared helpers for the audiocraft_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "../../include/audiocraft_b200.h"

// Thread-local last-error string (api.cu).
void acb_set_error(const char* fmt, ...);

#define ACB_CHECK_CUDA(expr)                                                                         \
    do {                                                                                             \
        cudaError_t e_ = (expr);                                                                     \
        if (e_ != cudaSuccess) {                                                                     \
            acb_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
            return ACB_ERR_CUDA;                                                                     \
        }                                                                                            \
    } while (0)

#define ACB_REQUIRE(cond, ...)            \
    do {                                  \
        if (!(cond)) {                    \
            acb_set_error(__VA_ARGS__);   \
            return ACB_ERR_INVALID;       \
        }                                 \
    } while (0)

#define ACB_LAUNCH_CHECK() ACB_CHECK_CUDA(cudaGetLastError())

#define ACB_TRY(expr) do { int rc_ = (expr); if (rc_ != ACB_OK) return rc_; } while (0)

static inline int acb_ceil_div(int a, int b) { return (a + b - 1) / b; }

// ELU(alpha=1) as torch computes it: x > 0 ? x : exp(x) - 1   (ATen elu kernel; not expm1)
// ELU: exp through ex2.approx (__expf, 2 instructions) instead of libm's expf (~10): absolute error ~1e-7 on (0, 1], the size of an
// fp32 rounding of the result.  Every golden stays index-exact and every layer test inside its tolerance; the slab staging of every
// encoder layer runs ELU per element, so the cheaper exp matters.  -DACB_PRECISE_ELU restores expf.
#ifdef ACB_PRECISE_ELU
__device__ __forceinline__ float acb_elu(float v) { return v > 0.f ? v : expf(v) - 1.f; }
#else
__device__ __forceinline__ float acb_elu(float v) { return v > 0.f ? v : __expf(v) - 1.f; }
#endif

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// 128-bit streaming load that does not allocate in L1 (weights / KV cache are read once per step).
__device__ __forceinline__ uint4 ld_stream_u4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
