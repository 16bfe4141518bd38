// Flash attention of the full-sequence forwards: the LM forward (lm_forward.cu) and the T5 encoder (t5.cu).
//
// softmax(scale * q k^T (+ bias)) v for head_dim 64, one CTA per (64-query tile, head, item), 4 warps of 16 query rows, K / V
// tiles of 64 keys in shared memory, scores and P.V on mma.sync m16n8k16 (fp16 operands, fp32 accumulation), online softmax
// in fp32.  Modes:
//   FA_CAUSAL (LM self attention): key tiles past the query tile are skipped and the diagonal tile is masked.
//   FA_CROSS  (LM cross attention): every key < Tk is attended, the condition's padded positions included.
//   FA_T5     (T5 encoder, bidirectional): scale 1 (T5 folds 1/sqrt(d) into its weights), plus the relative-position bias
//             rel_bias[bucket[j - i + Tq - 1]][h]; keys with key_mask[b][j] == 0 are excluded.  A query whose keys are all
//             excluded gets a zero output (finite, unlike a softmax over nothing).
// fp16 output into out [B * Tq][d] (FA_CAUSAL, FA_CROSS) or fp32 rounded to TF32 into out32 (FA_T5, the A operand of a TF32
// GEMM).
#pragma once
#include "common.cuh"
#include "lm_math.cuh"
#include "tma.cuh"
#include <math.h>

enum { FA_CAUSAL = 0, FA_CROSS = 1, FA_T5 = 2 };
constexpr int FA_BQ = 64, FA_BK = 64, FA_LD = 72;   // smem row pitch in halves: 144 B, conflict-free ldmatrix rows

struct FwdAttnParams {
    const __half* q; const __half* k; const __half* v;   // q [B][H][Tq][64], k / v [B][H][Tk][64]
    __half* out;
    int H, Tq, Tk, d;
    float scale;
    float* out32;              // FA_T5
    const float* rel_bias;     // FA_T5: [num_buckets][H]
    const int32_t* buckets;    // FA_T5: [2 Tq - 1], the bucket of relative position j - i at index j - i + Tq - 1 (Tk == Tq)
    const int64_t* key_mask;   // FA_T5: [B][Tk]
};

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}

template <int MODE>
__global__ void __launch_bounds__(128) lm_fwd_attn_kernel(FwdAttnParams p) {
    constexpr bool CAUSAL = MODE == FA_CAUSAL, T5 = MODE == FA_T5;
    __shared__ __align__(16) __half qs[FA_BQ * FA_LD];
    __shared__ __align__(16) __half ks[FA_BK * FA_LD];
    __shared__ __align__(16) __half vs[FA_BK * FA_LD];
    // FA_T5: the bias of relative position (k0 - q0) + r - (FA_BQ - 1) for r in [0, FA_BQ + FA_BK - 1), and 0 / -inf per key
    __shared__ float bias_s[T5 ? FA_BQ + FA_BK : 1];
    __shared__ float kmask_s[T5 ? FA_BK : 1];
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c4 = lane & 3;
    const int q0 = qt * FA_BQ;
    const __half* qg = p.q + ((size_t)b * p.H + h) * p.Tq * 64;
    const __half* kg = p.k + ((size_t)b * p.H + h) * p.Tk * 64;
    const __half* vg = p.v + ((size_t)b * p.H + h) * p.Tk * 64;

    for (int i = tid; i < FA_BQ * 8; i += 128) {   // rows past Tq are zero
        const int r = i >> 3, c = i & 7;
        uint4 val = make_uint4(0, 0, 0, 0);
        if (q0 + r < p.Tq) val = reinterpret_cast<const uint4*>(qg + (size_t)(q0 + r) * 64)[c];
        *reinterpret_cast<uint4*>(qs + r * FA_LD + c * 8) = val;
    }
    __syncthreads();
    uint32_t qf[4][4];   // A fragments of this warp's 16 query rows, 4 steps of 16 dims
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
        ldsm_x4(qf[kk], smem_u32(qs + (warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * FA_LD + kk * 16 + (lane >> 4) * 8));

    float o[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) o[nb][0] = o[nb][1] = o[nb][2] = o[nb][3] = 0.f;
    float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
    const int qa = q0 + warp * 16 + g;   // this thread's rows qa and qa + 8
    const int ktiles = (p.Tk + FA_BK - 1) / FA_BK;
    const int nkt = CAUSAL ? min(qt + 1, ktiles) : ktiles;

    for (int kt = 0; kt < nkt; ++kt) {
        const int k0 = kt * FA_BK;
        __syncthreads();   // every warp is done with the previous K / V tile
        for (int i = tid; i < FA_BK * 8; i += 128) {   // keys past Tk are zero (their scores are masked)
            const int r = i >> 3, c = i & 7;
            uint4 kv = make_uint4(0, 0, 0, 0), vv = kv;
            if (k0 + r < p.Tk) {
                kv = reinterpret_cast<const uint4*>(kg + (size_t)(k0 + r) * 64)[c];
                vv = reinterpret_cast<const uint4*>(vg + (size_t)(k0 + r) * 64)[c];
            }
            *reinterpret_cast<uint4*>(ks + r * FA_LD + c * 8) = kv;
            *reinterpret_cast<uint4*>(vs + r * FA_LD + c * 8) = vv;
        }
        if (T5) {
            for (int r = tid; r < FA_BQ + FA_BK - 1; r += 128) {   // positions outside [0, 2 Tq - 1) only meet masked scores
                const int idx = min(max(k0 - q0 + r - (FA_BQ - 1) + p.Tq - 1, 0), 2 * p.Tq - 2);
                bias_s[r] = p.rel_bias[(size_t)p.buckets[idx] * p.H + h];
            }
            if (tid < FA_BK) kmask_s[tid] = (k0 + tid < p.Tk && p.key_mask[(size_t)b * p.Tk + k0 + tid] != 0) ? 0.f : -INFINITY;
        }
        __syncthreads();

        float s[8][4];
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) {
            s[nb][0] = s[nb][1] = s[nb][2] = s[nb][3] = 0.f;
#pragma unroll
            for (int k2 = 0; k2 < 2; ++k2) {   // keys 8 nb .. 8 nb + 7, dims 32 k2 .. 32 k2 + 31
                uint32_t kb[4];
                ldsm_x4(kb, smem_u32(ks + (nb * 8 + (lane & 7)) * FA_LD + k2 * 32 + (lane >> 3) * 8));
                mma16816(s[nb], qf[2 * k2][0], qf[2 * k2][1], qf[2 * k2][2], qf[2 * k2][3], kb[0], kb[1]);
                mma16816(s[nb], qf[2 * k2 + 1][0], qf[2 * k2 + 1][1], qf[2 * k2 + 1][2], qf[2 * k2 + 1][3], kb[2], kb[3]);
            }
        }
        float mx[2] = {mrow[0], mrow[1]};
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int kl = nb * 8 + 2 * c4 + (i & 1), kidx = k0 + kl, qi = qa + 8 * (i >> 1);
                float v;
                if (T5) v = s[nb][i] + bias_s[kl - (qi - q0) + (FA_BQ - 1)] + kmask_s[kl];   // kmask_s is 0 or -inf
                else v = s[nb][i] * p.scale;
                if (kidx >= p.Tk || (CAUSAL && kidx > qi)) v = -INFINITY;
                s[nb][i] = v;
                mx[i >> 1] = fmaxf(mx[i >> 1], v);
            }
        float corr[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            corr[r] = mrow[r] == -INFINITY ? 0.f : __expf(mrow[r] - mx[r]);
            mrow[r] = mx[r];
            lrow[r] *= corr[r];
        }
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float mr = mx[i >> 1];
                const float pw = mr == -INFINITY ? 0.f : __expf(s[nb][i] - mr);
                s[nb][i] = pw;
                lrow[i >> 1] += pw;
                o[nb][i] *= corr[i >> 1];
            }
#pragma unroll
        for (int j = 0; j < 4; ++j) {   // keys 16 j .. 16 j + 15: P as the A operand straight from the score registers
            const uint32_t a0 = pack_half2(s[2 * j][0], s[2 * j][1]), a1 = pack_half2(s[2 * j][2], s[2 * j][3]);
            const uint32_t a2 = pack_half2(s[2 * j + 1][0], s[2 * j + 1][1]), a3 = pack_half2(s[2 * j + 1][2], s[2 * j + 1][3]);
#pragma unroll
            for (int nb2 = 0; nb2 < 4; ++nb2) {   // dims 16 nb2 .. 16 nb2 + 15: V transposed by ldmatrix
                uint32_t vb[4];
                ldsm_x4_trans(vb, smem_u32(vs + (16 * j + (lane & 7) + ((lane >> 3) & 1) * 8) * FA_LD + nb2 * 16 + (lane >> 4) * 8));
                mma16816(o[2 * nb2], a0, a1, a2, a3, vb[0], vb[1]);
                mma16816(o[2 * nb2 + 1], a0, a1, a2, a3, vb[2], vb[3]);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 1);
        lrow[r] += __shfl_xor_sync(0xffffffffu, lrow[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int qi = qa + 8 * r;
        if (qi >= p.Tq) continue;
        if (T5) {
            const float inv = lrow[r] > 0.f ? 1.f / lrow[r] : 0.f;   // every key masked: o is 0, keep it 0
            float* dst = p.out32 + ((size_t)b * p.Tq + qi) * p.d + h * 64 + 2 * c4;
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
                *reinterpret_cast<float2*>(dst + nb * 8) = make_float2(tf32_round(o[nb][2 * r] * inv), tf32_round(o[nb][2 * r + 1] * inv));
        } else {
            const float inv = 1.f / lrow[r];
            __half* dst = p.out + ((size_t)b * p.Tq + qi) * p.d + h * 64 + 2 * c4;
#pragma unroll
            for (int nb = 0; nb < 8; ++nb)
                *reinterpret_cast<__half2*>(dst + nb * 8) = __floats2half2_rn(o[nb][2 * r] * inv, o[nb][2 * r + 1] * inv);
        }
    }
}
