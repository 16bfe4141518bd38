// mbarrier and tiled-TMA helpers shared by the LM decode step (lm.cu) and the full-sequence forwards (fwd_gemm.cuh).
#pragma once
#include <cudaTypedefs.h>   // CUtensorMap, PFN_cuTensorMapEncodeTiled: types only, the entry point is looked up at run time
#include <stdint.h>
#include "common.cuh"

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    do {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}

// 2-D tiled TMA load of box (c0 = inner coordinate, c1 = outer) into shared memory, completion on an mbarrier.
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

static PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &f, 12000, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
    }
    return fn;
}

// Tensor map of a row-major [outer][inner] matrix of `elem_bytes`-byte elements read in boxes of box_outer rows x one
// swizzle row (box_inner elements), 128-byte swizzled unless `swizzle` says otherwise; boxes past either edge are zero-filled.
static int encode_map_typed(CUtensorMap* m, const void* base, int inner, int outer, int box_outer, CUtensorMapDataType dt,
                            int elem_bytes, int box_inner, const char* what,
                            CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
    PFN_cuTensorMapEncodeTiled_v12000 fn = tensor_map_encoder();
    ACB_REQUIRE(fn, "lm: cuTensorMapEncodeTiled is not available from the CUDA driver");
    cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer}, strides[1] = {(cuuint64_t)inner * elem_bytes};
    cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer}, es[2] = {1, 1};
    const CUresult r = fn(m, dt, 2, const_cast<void*>(base), dims, strides, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    ACB_REQUIRE(r == CUDA_SUCCESS, "lm: cuTensorMapEncodeTiled failed (%d) for a [%d][%d] %s matrix", (int)r, outer, inner, what);
    return ACB_OK;
}

// fp16 matrix, boxes of 64 elements
constexpr int TMA_BOX_K = 64;
static int encode_map(CUtensorMap* m, const void* base, int inner, int outer, int box_outer) {
    return encode_map_typed(m, base, inner, outer, box_outer, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, TMA_BOX_K, "fp16");
}
// fp32 matrix (a TF32 wgmma operand), boxes of 32 elements
constexpr int TMA_BOX_K_F32 = 32;
static int encode_map_f32(CUtensorMap* m, const void* base, int inner, int outer, int box_outer) {
    return encode_map_typed(m, base, inner, outer, box_outer, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, TMA_BOX_K_F32, "fp32");
}
// e4m3 matrix (FP8 weights of the wide decode GEMM), boxes of 64 bytes in the 64-byte swizzle (lm_gemm_wide_fp8_kernel)
static int encode_map_u8(CUtensorMap* m, const void* base, int inner, int outer, int box_outer) {
    return encode_map_typed(m, base, inner, outer, box_outer, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, 64, "e4m3",
                            CU_TENSOR_MAP_SWIZZLE_64B);
}
