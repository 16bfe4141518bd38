// Tiled wgmma GEMM of the full-sequence forwards: the LM forward (lm_forward.cu, fp16 operands) and the T5 encoder (t5.cu,
// fp32 operands on the TF32 tensor pipe).
//
// C[M][N] = A[M][K] . W[N][K]^T, A the activations, W a stacked weight matrix [L * N][K] (the layer is the row offset
// w_row0).  CTA = 128 x 128 output tile, 3 warpgroups: warpgroup 0 is the producer (one thread issues the TMA loads of
// 128-byte K chunks into a FG_STAGES-deep ring), warpgroups 1 and 2 each own 64 rows of the tile and issue m64n128 wgmmas.
// One chunk is 64 fp16 elements (4 k16 steps) or 32 fp32 elements (4 k8 TF32 steps); either way a step advances the
// descriptors by 32 bytes, so both operand types share the ring, the barriers and the epilogue.  K, M and N tails: TMA
// zero-fills boxes past the matrix edges and the epilogue masks rows >= M and columns >= N.  No split-K: every output
// element is summed by one CTA in one fixed order, so an item's results do not depend on the batch it is in, and the
// residual add is a plain read-modify-write.
#pragma once
#include "common.cuh"
#include "lm_math.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

enum { FE_QKV = 0, FE_QKV_ROPE = 1, FE_CKV = 2, FE_RESID = 3, FE_GELU = 4, FE_LOGITS = 5, FE_RELU = 6, FE_PROJ = 7 };
constexpr int FG_BM = 128, FG_BN = 128, FG_STAGES = 5, FG_THREADS = 384;
constexpr int FG_TILE = 128 * 128;             // bytes of one 128-row box of 128-byte rows
constexpr int FG_STAGE = 2 * FG_TILE;          // A box + W box
constexpr int FG_SMEM = FG_STAGES * FG_STAGE + 1024 + 2 * FG_STAGES * 8;   // ring (1024-aligned) + full / empty barriers
static_assert(FG_TILE == 128 * TMA_BOX_K * 2 && FG_TILE == 128 * TMA_BOX_K_F32 * 4, "one box row is one 128-byte swizzle row");

struct FwdGemmParams {
    int M, N, K, w_row0;
    int T;              // token rows per item (P + S); FE_CKV: text positions per item
    int P, S, H, d;     // prefix length, sequence length, heads, model dim
    __half* q; __half* k; __half* v;   // FE_QKV(_ROPE): [B][H][T][64] each (q alone when N == d); FE_CKV: k, v [B][H][text][64]
    float* x;           // FE_RESID: [M][d]
    __half* f16;        // FE_GELU: [M][N]
    float* logits;      // FE_LOGITS: [B][N / card][S][card]
    int card;
    float pos_scale;
    const float* rope_freq;   // FE_QKV_ROPE: [32]
    float* f32;               // FE_RELU (rounded to TF32: the next GEMM's operand), FE_PROJ: [M][N]
    const float* bias;        // FE_PROJ: [N]
    const int64_t* mask;      // FE_PROJ: [M] (0 or 1 per token row)
};

template <int EPI>
__device__ __forceinline__ void fwd_store(const FwdGemmParams& p, int m, int b, int t, int n, float v0, float v1) {
    if (EPI == FE_QKV || EPI == FE_QKV_ROPE || EPI == FE_CKV) {
        const int which = n >= 2 * p.d ? 2 : (n >= p.d ? 1 : 0), nn = n - which * p.d, dd = nn & 63;
        if (EPI == FE_QKV_ROPE && which < 2) {
            // RotaryEmbedding.rotate_qk (modules/rope.py:84-125) as rope_rotate of the decode step: the pair (dd, dd + 1) is
            // (v0, v1), rotated by t * rope_freq[dd / 2] in fp32 from fp16-rounded values and blended with pos_scale
            const float re = half_round(v0), im = half_round(v1);
            float sn, cs;
            sincosf((float)t * p.rope_freq[dd >> 1], &sn, &cs);
            const float rr = cs * p.pos_scale + (1.f - p.pos_scale), ri = sn * p.pos_scale;
            v0 = re * rr - im * ri;
            v1 = re * ri + im * rr;
        }
        __half* dst = EPI == FE_CKV ? (which ? p.v : p.k) : (which == 0 ? p.q : (which == 1 ? p.k : p.v));
        *reinterpret_cast<__half2*>(dst + (((size_t)b * p.H + (nn >> 6)) * p.T + t) * 64 + dd) = __floats2half2_rn(v0, v1);
    } else if (EPI == FE_RESID) {
        float2* px = reinterpret_cast<float2*>(p.x + (size_t)m * p.d + n);
        float2 xv = *px;
        xv.x += v0;
        xv.y += v1;
        *px = xv;
    } else if (EPI == FE_GELU) {
        *reinterpret_cast<__half2*>(p.f16 + (size_t)m * p.N + n) =
            __floats2half2_rn(gelu_erf(half_round(v0)), gelu_erf(half_round(v1)));
    } else if (EPI == FE_RELU) {
        *reinterpret_cast<float2*>(p.f32 + (size_t)m * p.N + n) = make_float2(tf32_round(fmaxf(v0, 0.f)), tf32_round(fmaxf(v1, 0.f)));
    } else if (EPI == FE_PROJ) {   // (acc + bias) * mask: masked token rows are exact zeros (acc is finite)
        const float mk = (float)p.mask[m];
        *reinterpret_cast<float2*>(p.f32 + (size_t)m * p.N + n) = make_float2((v0 + p.bias[n]) * mk, (v1 + p.bias[n + 1]) * mk);
    } else {   // FE_LOGITS: sequence positions only (the prefix's logits are dropped, lm.py:264-266)
        if (t < p.P) return;
        const int kq = n / p.card, c = n - kq * p.card;
        *reinterpret_cast<float2*>(p.logits + (((size_t)b * (p.N / p.card) + kq) * p.S + (t - p.P)) * p.card + c) =
            make_float2(v0, v1);
    }
}

// TF32: fp32 operands (tensor maps from encode_map_f32), m64n128k8; otherwise fp16 operands (encode_map), m64n128k16.
template <bool TF32, int EPI>
__global__ void __launch_bounds__(FG_THREADS, 1) lm_fwd_gemm_kernel(const __grid_constant__ CUtensorMap amap,
                                                                    const __grid_constant__ CUtensorMap wmap, FwdGemmParams p) {
    constexpr int BOX_K = TF32 ? TMA_BOX_K_F32 : TMA_BOX_K;   // elements of one 128-byte chunk
    extern __shared__ unsigned char fg_raw[];
    unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(fg_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(sm + FG_STAGES * FG_STAGE);
    uint64_t* empty = full + FG_STAGES;
    const int tid = threadIdx.x, wg = tid >> 7;
    const int n0 = blockIdx.x * FG_BN, m0 = blockIdx.y * FG_BM;
    const int nch = (p.K + BOX_K - 1) / BOX_K;

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < FG_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 2 * 128);   // every consumer thread releases the stage
        }
    }
    __syncthreads();
    if (wg == 0) {   // producer
        if (tid == 0) {
            for (int c = 0; c < nch; ++c) {
                const int s = c % FG_STAGES;
                if (c >= FG_STAGES) mbar_wait(&empty[s], (uint32_t)(c / FG_STAGES - 1) & 1u);
                unsigned char* st = sm + s * FG_STAGE;
                mbar_expect_tx(&full[s], (uint32_t)FG_STAGE);   // zero-filled bytes count too
                tma_load_2d(st, &amap, c * BOX_K, m0, &full[s]);
                tma_load_2d(st + FG_TILE, &wmap, c * BOX_K, p.w_row0 + n0, &full[s]);
            }
        }
        return;   // the consumers wait for every load before the CTA can exit
    }

    const int cw = wg - 1;   // rows [64 cw, 64 cw + 64) of the tile
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int c = 0; c < nch; ++c) {
        const int s = c % FG_STAGES;
        mbar_wait(&full[s], (uint32_t)(c / FG_STAGES) & 1u);
        const uint32_t a = smem_u32(sm + s * FG_STAGE) + cw * 64 * 128, b = smem_u32(sm + s * FG_STAGE + FG_TILE);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {   // a K step (16 fp16 or 8 fp32 elements) advances the start address by 32 bytes
            if (TF32) wgmma_tf32<128>(acc, wgmma_desc_sw128(a + 32 * kk), wgmma_desc_sw128(b + 32 * kk), 1u);
            else wgmma_f16<128>(acc, wgmma_desc_sw128(a + 32 * kk), wgmma_desc_sw128(b + 32 * kk), 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the MMAs of chunk c - 1 have finished reading their stage
        if (c > 0) mbar_arrive(&empty[(c - 1) % FG_STAGES]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);

    // thread (warp w of the warpgroup, lane l) holds acc[4j + i] at row 16 w + l / 4 + 8 (i / 2), column 8 j + 2 (l % 4) + (i % 2)
    const int warp = (tid >> 5) & 3, lane = tid & 31;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int m = m0 + 64 * cw + 16 * warp + (lane >> 2) + 8 * hr;
        if (m >= p.M) continue;
        const int b = m / p.T, t = m - b * p.T;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int n = n0 + 8 * j + 2 * (lane & 3);
            if (n < p.N) fwd_store<EPI>(p, m, b, t, n, acc[4 * j + 2 * hr], acc[4 * j + 2 * hr + 1]);
        }
    }
}

// Launches one GEMM; am / wm are tensor maps of the operand type TF32 selects, with FG_BM / FG_BN-row boxes.
template <int EPI, bool TF32 = false>
static int fwd_gemm(const CUtensorMap& am, const CUtensorMap& wm, const FwdGemmParams& p, cudaStream_t s) {
    ACB_CHECK_CUDA(cudaFuncSetAttribute(lm_fwd_gemm_kernel<TF32, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, FG_SMEM));
    const dim3 grid(acb_ceil_div(p.N, FG_BN), acb_ceil_div(p.M, FG_BM));
    lm_fwd_gemm_kernel<TF32, EPI><<<grid, FG_THREADS, FG_SMEM, s>>>(am, wm, p);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}
