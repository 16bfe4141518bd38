// MusicGen LM full-sequence forward for H100 (sm_90a): LMModel.forward over whole sequences (audiocraft/models/lm.py:221-268),
// the computation behind LMModel.compute_predictions (lm.py:270-321), i.e. scoring codes under the LM.
//
// Unlike the decode step (lm.cu), which streams every weight once per generated position and is bound by HBM bandwidth, the
// forward multiplies the whole token matrix (M = batch * (prefix + seq_len) rows) by each weight once and is compute-bound:
//   * every matrix product is one tiled wgmma GEMM (lm_fwd_gemm_kernel): 128 x 128 output tiles, both operands K-major in
//     the 128-byte swizzle that tiled TMA writes into an mbarrier ring, one producer warp issuing the loads and two consumer
//     warpgroups issuing the MMAs.  No split-K: every output element is summed by one CTA in one fixed order, so an item's
//     results do not depend on the batch it is in, and the residual add is a plain read-modify-write.
//   * the epilogue of each GEMM writes its consumer's layout directly: q / k / v head-major (with rotary positions), the
//     condition's cross K / V, x += acc, GELU to fp16, or fp32 logits of the sequence positions.
//   * attention is a flash-attention kernel on mma.sync (lm_fwd_attn_kernel): causal for self attention, every text position
//     (padding included, as the reference does) for cross attention.
// fp16 GEMM operands, fp32 accumulation, fp32 residual stream and LayerNorm, as in the decode step (DESIGN.md section 2).
// The kernels restate the element arithmetic of the decode kernels (embedding + sin term, LayerNorm, GELU, rotary) so that
// forward and decode agree.  Nothing here touches a decode handle: the call is stateless and graph-capturable.
#include "common.cuh"
#include "lm_math.cuh"
#include "tma.cuh"
#include "wgmma.cuh"
#include <math.h>

// ------------------------------------------------------------------------------------------------ embedding
// x[m] for token row m = b * T + t (T = P + S): the condition prefix (rounded to fp16 like the reference's autocast
// output_proj) for t < P, else sum_k emb_k[seq[b][k][t - P]]; plus pos_scale * [cos(t / f_i), sin(t / f_i)] when sin_pos.
// The same element arithmetic as lm_embed_kernel / lm_embed_prefix_kernel of the decode step.
__global__ void __launch_bounds__(256) lm_fwd_embed_kernel(const __half* __restrict__ emb, const float* __restrict__ inv_freq,
                                                           const int64_t* __restrict__ seq, const float* __restrict__ prefix,
                                                           float* __restrict__ x, int d, int n_q, int card, int T, int P, int S,
                                                           float pos_scale, bool sin_pos) {
    const int m = blockIdx.x, b = m / T, t = m - b * T;
    __shared__ int tok[16];
    if (t >= P && threadIdx.x < n_q) tok[threadIdx.x] = (int)seq[((size_t)b * n_q + threadIdx.x) * S + (t - P)];
    __syncthreads();
    const int half_d = d >> 1;
    for (int i = threadIdx.x; i < d; i += 256) {
        float v = 0.f;
        if (t < P) v = half_round(prefix[((size_t)b * P + t) * d + i]);
        else
            for (int k = 0; k < n_q; ++k) v += __half2float(emb[((size_t)k * (card + 1) + tok[k]) * d + i]);
        if (sin_pos) {
            const int j = i < half_d ? i : i - half_d;
            const float phase = (float)t / inv_freq[j];
            v += pos_scale * (i < half_d ? cosf(phase) : sinf(phase));
        }
        x[(size_t)m * d + i] = v;
    }
}

// ------------------------------------------------------------------------------------------------ LayerNorm
// out[m] = LayerNorm(x[m]) * gamma + beta (eps 1e-5, fp32 statistics), rounded to fp16: lm_ln_kernel's arithmetic without
// the split-K partial sums (the forward GEMMs add into x themselves).  One CTA per row, one float4 per thread (d <= 2048).
constexpr int FLN_THREADS = 512;
__global__ void __launch_bounds__(FLN_THREADS) lm_fwd_ln_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                                const float* __restrict__ beta, __half* __restrict__ out, int d) {
    __shared__ float red[2][32];
    const int r = blockIdx.x, i = threadIdx.x;
    const bool live = i < (d >> 2);
    float4 gm = make_float4(0.f, 0.f, 0.f, 0.f), bt = gm, a = gm;
    if (live) {
        gm = reinterpret_cast<const float4*>(gamma)[i];
        bt = reinterpret_cast<const float4*>(beta)[i];
        a = reinterpret_cast<const float4*>(x + (size_t)r * d)[i];
    }
    const float mean = block_sum((a.x + a.y) + (a.z + a.w), red[0]) / d;
    float q = 0.f;
    if (live) {
        const float cx = a.x - mean, cy = a.y - mean, cz = a.z - mean, cw = a.w - mean;
        q = fmaf(cx, cx, q); q = fmaf(cy, cy, q); q = fmaf(cz, cz, q); q = fmaf(cw, cw, q);
    }
    const float rstd = 1.f / sqrtf(block_sum(q, red[1]) / d + 1e-5f);
    if (live) {
        __half2 lo = __floats2half2_rn((a.x - mean) * rstd * gm.x + bt.x, (a.y - mean) * rstd * gm.y + bt.y);
        __half2 hi = __floats2half2_rn((a.z - mean) * rstd * gm.z + bt.z, (a.w - mean) * rstd * gm.w + bt.w);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t*>(&lo);
        pk.y = *reinterpret_cast<uint32_t*>(&hi);
        reinterpret_cast<uint2*>(out + (size_t)r * d)[i] = pk;
    }
}

__global__ void lm_fwd_f32_to_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = __float2half_rn(src[i]);
}

// ------------------------------------------------------------------------------------------------ tiled GEMM
// C[M][N] = A[M][K] . W[N][K]^T, A the fp16 activations, W a stacked weight matrix [L * N][K] (the layer is the row offset
// w_row0).  CTA = 128 x 128 output tile, 3 warpgroups: warpgroup 0 is the producer (one thread issues the TMA loads of 64-element
// K chunks into a FG_STAGES-deep ring), warpgroups 1 and 2 each own 64 rows of the tile and issue m64n128k16 wgmmas.  K, M and
// N tails: TMA zero-fills boxes past the matrix edges and the epilogue masks rows >= M and columns >= N.
enum { FE_QKV = 0, FE_QKV_ROPE = 1, FE_CKV = 2, FE_RESID = 3, FE_GELU = 4, FE_LOGITS = 5 };
constexpr int FG_BM = 128, FG_BN = 128, FG_STAGES = 5, FG_THREADS = 384;
constexpr int FG_TILE = 128 * TMA_BOX_K * 2;   // bytes of one 128-row box
constexpr int FG_STAGE = 2 * FG_TILE;          // A box + W box
constexpr int FG_SMEM = FG_STAGES * FG_STAGE + 1024 + 2 * FG_STAGES * 8;   // ring (1024-aligned) + full / empty barriers

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
    } else {   // FE_LOGITS: sequence positions only (the prefix's logits are dropped, lm.py:264-266)
        if (t < p.P) return;
        const int kq = n / p.card, c = n - kq * p.card;
        *reinterpret_cast<float2*>(p.logits + (((size_t)b * (p.N / p.card) + kq) * p.S + (t - p.P)) * p.card + c) =
            make_float2(v0, v1);
    }
}

template <int EPI>
__global__ void __launch_bounds__(FG_THREADS, 1) lm_fwd_gemm_kernel(const __grid_constant__ CUtensorMap amap,
                                                                    const __grid_constant__ CUtensorMap wmap, FwdGemmParams p) {
    extern __shared__ unsigned char fg_raw[];
    unsigned char* sm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(fg_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(sm + FG_STAGES * FG_STAGE);
    uint64_t* empty = full + FG_STAGES;
    const int tid = threadIdx.x, wg = tid >> 7;
    const int n0 = blockIdx.x * FG_BN, m0 = blockIdx.y * FG_BM;
    const int nch = (p.K + TMA_BOX_K - 1) / TMA_BOX_K;

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
                tma_load_2d(st, &amap, c * TMA_BOX_K, m0, &full[s]);
                tma_load_2d(st + FG_TILE, &wmap, c * TMA_BOX_K, p.w_row0 + n0, &full[s]);
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
        for (int kk = 0; kk < TMA_BOX_K / 16; ++kk)   // a 16-element K step advances the start address by 32 bytes
            wgmma_f16<128>(acc, wgmma_desc_sw128(a + 32 * kk), wgmma_desc_sw128(b + 32 * kk), 1u);
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

// ------------------------------------------------------------------------------------------------ flash attention
// softmax(q k^T / 8) v for head_dim 64, one CTA per (64-query tile, head, item), 4 warps of 16 query rows, K / V tiles of 64
// keys in shared memory, scores and P.V on mma.sync m16n8k16 (fp16 operands, fp32 accumulation), online softmax in fp32.
// CAUSAL (self attention): key tiles past the query tile are skipped and the diagonal tile is masked.  Otherwise (cross
// attention) every key < Tk is attended, the condition's padded positions included.  Output fp16 into out [B * Tq][d].
constexpr int FA_BQ = 64, FA_BK = 64, FA_LD = 72;   // smem row pitch in halves: 144 B, conflict-free ldmatrix rows

struct FwdAttnParams {
    const __half* q; const __half* k; const __half* v;   // q [B][H][Tq][64], k / v [B][H][Tk][64]
    __half* out;
    int H, Tq, Tk, d;
    float scale;
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

template <bool CAUSAL>
__global__ void __launch_bounds__(128) lm_fwd_attn_kernel(FwdAttnParams p) {
    __shared__ __align__(16) __half qs[FA_BQ * FA_LD];
    __shared__ __align__(16) __half ks[FA_BK * FA_LD];
    __shared__ __align__(16) __half vs[FA_BK * FA_LD];
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
                const int kidx = k0 + nb * 8 + 2 * c4 + (i & 1), qi = qa + 8 * (i >> 1);
                float v = s[nb][i] * p.scale;
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
        const float inv = 1.f / lrow[r];
        __half* dst = p.out + ((size_t)b * p.Tq + qi) * p.d + h * 64 + 2 * c4;
#pragma unroll
        for (int nb = 0; nb < 8; ++nb)
            *reinterpret_cast<__half2*>(dst + nb * 8) = __floats2half2_rn(o[nb][2 * r] * inv, o[nb][2 * r + 1] * inv);
    }
}

// ------------------------------------------------------------------------------------------------ host side
namespace {
struct FwdLayout {
    size_t x, h16, q, k, v, a16, f16, c16, ck, cv, total;
};

size_t fwd_take(size_t* off, size_t bytes) {
    const size_t at = *off;
    *off += (bytes + 255) / 256 * 256;
    return at;
}

// Validates the shapes (no pointer is touched) and lays out the workspace.
int fwd_layout(const acb_lm_config* c, int batch, int prefix_len, int seq_len, int text_len, FwdLayout* L) {
    ACB_REQUIRE(c, "acb_lm_forward: null config");
    ACB_REQUIRE(c->dim >= 64 && c->dim % 64 == 0 && c->dim == c->num_heads * 64 && c->dim <= 4 * FLN_THREADS,
                "acb_lm_forward: dim %d / heads %d: head_dim must be 64 and dim <= %d", c->dim, c->num_heads, 4 * FLN_THREADS);
    ACB_REQUIRE(c->num_layers >= 1, "acb_lm_forward: num_layers %d", c->num_layers);
    ACB_REQUIRE(c->ffn_dim >= 8 && c->ffn_dim % 8 == 0, "acb_lm_forward: ffn_dim %d must be a positive multiple of 8", c->ffn_dim);
    ACB_REQUIRE(c->n_q >= 1 && c->n_q <= 16 && c->card >= 2 && c->card % 2 == 0,
                "acb_lm_forward: n_q %d must be in [1, 16] and card %d even", c->n_q, c->card);
    ACB_REQUIRE(c->positional_embedding >= 0 && c->positional_embedding <= 2, "acb_lm_forward: positional_embedding %d not in [0,2]",
                c->positional_embedding);
    ACB_REQUIRE(batch >= 1 && seq_len >= 1 && prefix_len >= 0 && text_len >= 0,
                "acb_lm_forward: batch %d, seq_len %d, prefix_len %d, text_len %d", batch, seq_len, prefix_len, text_len);
    ACB_REQUIRE(!c->cross_attention || text_len >= 1, "acb_lm_forward: the model has cross attention, text_len must be >= 1");
    const int64_t T = (int64_t)prefix_len + seq_len, M = (int64_t)batch * T;
    // the GEMM grid's y dimension is one CTA per FG_BM rows, the attention grid's z dimension one CTA per item (65535 each)
    constexpr int64_t max_rows = (int64_t)65535 * FG_BM;
    ACB_REQUIRE(M <= max_rows && batch <= 65535 && (int64_t)batch * text_len <= max_rows,
                "acb_lm_forward: %lld token rows, %lld condition rows (batch %d): at most %lld rows and 65535 items",
                (long long)M, (long long)batch * text_len, batch, (long long)max_rows);
    const size_t d = c->dim, h = 2, Mz = (size_t)M, Mt = (size_t)batch * (c->cross_attention ? text_len : 0);
    size_t off = 0;
    L->x = fwd_take(&off, Mz * d * 4);
    L->h16 = fwd_take(&off, Mz * d * h);
    L->q = fwd_take(&off, Mz * d * h);
    L->k = fwd_take(&off, Mz * d * h);
    L->v = fwd_take(&off, Mz * d * h);
    L->a16 = fwd_take(&off, Mz * d * h);
    L->f16 = fwd_take(&off, Mz * (size_t)c->ffn_dim * h);
    L->c16 = fwd_take(&off, Mt * d * h);
    L->ck = fwd_take(&off, Mt * d * h);
    L->cv = fwd_take(&off, Mt * d * h);
    L->total = off;
    return ACB_OK;
}

template <int EPI>
int fwd_gemm(const CUtensorMap& am, const CUtensorMap& wm, const FwdGemmParams& p, cudaStream_t s) {
    ACB_CHECK_CUDA(cudaFuncSetAttribute(lm_fwd_gemm_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, FG_SMEM));
    const dim3 grid(acb_ceil_div(p.N, FG_BN), acb_ceil_div(p.M, FG_BM));
    lm_fwd_gemm_kernel<EPI><<<grid, FG_THREADS, FG_SMEM, s>>>(am, wm, p);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

int fwd_attn(bool causal, const FwdAttnParams& a, int batch, cudaStream_t s) {
    const dim3 grid(acb_ceil_div(a.Tq, FA_BQ), a.H, batch);
    if (causal) lm_fwd_attn_kernel<true><<<grid, 128, 0, s>>>(a);
    else lm_fwd_attn_kernel<false><<<grid, 128, 0, s>>>(a);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}
}   // namespace

extern "C" int64_t acb_lm_forward_workspace_bytes(const acb_lm_config* cfg, int batch, int prefix_len, int seq_len, int text_len) {
    FwdLayout L;
    const int rc = fwd_layout(cfg, batch, prefix_len, seq_len, text_len, &L);
    return rc != ACB_OK ? (int64_t)rc : (int64_t)L.total;
}

extern "C" int acb_lm_forward(const acb_lm_config* cfg, const acb_lm_weights* w, const int64_t* seq, const float* cross,
                              const float* prefix, int batch, int prefix_len, int seq_len, int text_len, float* logits,
                              void* workspace, int64_t workspace_bytes, void* stream) {
    FwdLayout L;
    ACB_TRY(fwd_layout(cfg, batch, prefix_len, seq_len, text_len, &L));
    const acb_lm_config& c = *cfg;
    const bool has_cross = c.cross_attention != 0, rope = c.positional_embedding != 0, sin_pos = c.positional_embedding != 1;
    ACB_REQUIRE(w && seq && logits && workspace, "acb_lm_forward: null weights, sequence, logits or workspace");
    ACB_REQUIRE(w->emb && w->w_qkv && w->w_o && w->w_ff1 && w->w_ff2 && w->ln && w->out_norm && w->heads &&
                (!sin_pos || w->inv_freq) && (!rope || w->rope_freq) && (!has_cross || (w->w_cq && w->w_ckv && w->w_co)),
                "acb_lm_forward: a weight the config needs is NULL");
    ACB_REQUIRE((prefix_len > 0) == (prefix != nullptr), "acb_lm_forward: prefix must be given exactly when prefix_len > 0 (%d)",
                prefix_len);
    ACB_REQUIRE(has_cross == (cross != nullptr), "acb_lm_forward: the condition tensor must be given exactly when the model has "
                "cross attention (the reference asserts the same, transformer.py:553-556)");
    ACB_REQUIRE(workspace_bytes >= (int64_t)L.total, "acb_lm_forward: workspace of %lld bytes < %lld needed",
                (long long)workspace_bytes, (long long)L.total);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    float* x = reinterpret_cast<float*>(ws + L.x);
    __half *h16 = reinterpret_cast<__half*>(ws + L.h16), *q = reinterpret_cast<__half*>(ws + L.q);
    __half *k = reinterpret_cast<__half*>(ws + L.k), *v = reinterpret_cast<__half*>(ws + L.v);
    __half *a16 = reinterpret_cast<__half*>(ws + L.a16), *f16 = reinterpret_cast<__half*>(ws + L.f16);
    __half *c16 = reinterpret_cast<__half*>(ws + L.c16), *ck = reinterpret_cast<__half*>(ws + L.ck);
    __half* cv = reinterpret_cast<__half*>(ws + L.cv);
    const int d = c.dim, ffn = c.ffn_dim, H = c.num_heads, NL = c.num_layers, T = prefix_len + seq_len, M = batch * T;
    const int Mt = has_cross ? batch * text_len : 0, NV = c.n_q * c.card;

    // tensor maps: activations [rows][K] and stacked weights [L * N][K], 128-row boxes
    CUtensorMap m_h16, m_a16, m_f16, m_c16, m_qkv, m_o, m_cq, m_ckv, m_co, m_ff1, m_ff2, m_heads;
    ACB_TRY(encode_map(&m_h16, h16, d, M, FG_BM));
    ACB_TRY(encode_map(&m_a16, a16, d, M, FG_BM));
    ACB_TRY(encode_map(&m_f16, f16, ffn, M, FG_BM));
    ACB_TRY(encode_map(&m_qkv, w->w_qkv, d, NL * 3 * d, FG_BN));
    ACB_TRY(encode_map(&m_o, w->w_o, d, NL * d, FG_BN));
    ACB_TRY(encode_map(&m_ff1, w->w_ff1, d, NL * ffn, FG_BN));
    ACB_TRY(encode_map(&m_ff2, w->w_ff2, ffn, NL * d, FG_BN));
    ACB_TRY(encode_map(&m_heads, w->heads, d, NV, FG_BN));
    if (has_cross) {
        ACB_TRY(encode_map(&m_c16, c16, d, Mt, FG_BM));
        ACB_TRY(encode_map(&m_cq, w->w_cq, d, NL * d, FG_BN));
        ACB_TRY(encode_map(&m_ckv, w->w_ckv, d, NL * 2 * d, FG_BN));
        ACB_TRY(encode_map(&m_co, w->w_co, d, NL * d, FG_BN));
    }

    lm_fwd_embed_kernel<<<M, 256, 0, s>>>((const __half*)w->emb, w->inv_freq, seq, prefix, x, d, c.n_q, c.card, T, prefix_len,
                                          seq_len, c.pos_scale, sin_pos);
    ACB_LAUNCH_CHECK();
    if (has_cross) {
        const size_t n = (size_t)Mt * d;
        lm_fwd_f32_to_f16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(cross, c16, n);
        ACB_LAUNCH_CHECK();
    }
    FwdGemmParams base{};
    base.M = M; base.K = d; base.T = T; base.P = prefix_len; base.S = seq_len; base.H = H; base.d = d;
    base.q = q; base.k = k; base.v = v; base.x = x; base.f16 = f16; base.logits = logits; base.card = c.card;
    base.pos_scale = c.pos_scale; base.rope_freq = w->rope_freq;
    const float scale = 1.0f / sqrtf(64.f);
    auto ln = [&](const float* gamma, const float* beta) -> int {
        lm_fwd_ln_kernel<<<M, FLN_THREADS, 0, s>>>(x, gamma, beta, h16, d);
        ACB_LAUNCH_CHECK();
        return ACB_OK;
    };
    for (int l = 0; l < NL; ++l) {
        const float* lnw = w->ln + (size_t)l * 6 * d;
        // self attention
        ACB_TRY(ln(lnw, lnw + d));
        FwdGemmParams p = base;
        p.N = 3 * d; p.w_row0 = l * 3 * d;
        ACB_TRY(rope ? fwd_gemm<FE_QKV_ROPE>(m_h16, m_qkv, p, s) : fwd_gemm<FE_QKV>(m_h16, m_qkv, p, s));
        ACB_TRY(fwd_attn(true, FwdAttnParams{q, k, v, a16, H, T, T, d, scale}, batch, s));
        p = base;
        p.N = d; p.w_row0 = l * d;
        ACB_TRY(fwd_gemm<FE_RESID>(m_a16, m_o, p, s));
        // cross attention: queries of the tokens, K / V of the condition (this layer's)
        if (has_cross) {
            ACB_TRY(ln(lnw + 2 * d, lnw + 3 * d));
            p = base;
            p.N = d; p.w_row0 = l * d;   // q alone: every column is in the q block
            ACB_TRY(fwd_gemm<FE_QKV>(m_h16, m_cq, p, s));
            p = base;
            p.M = Mt; p.N = 2 * d; p.w_row0 = l * 2 * d; p.T = text_len; p.k = ck; p.v = cv;
            ACB_TRY(fwd_gemm<FE_CKV>(m_c16, m_ckv, p, s));
            ACB_TRY(fwd_attn(false, FwdAttnParams{q, ck, cv, a16, H, T, text_len, d, scale}, batch, s));
            p = base;
            p.N = d; p.w_row0 = l * d;
            ACB_TRY(fwd_gemm<FE_RESID>(m_a16, m_co, p, s));
        }
        // feed forward
        ACB_TRY(ln(lnw + 4 * d, lnw + 5 * d));
        p = base;
        p.N = ffn; p.w_row0 = l * ffn;
        ACB_TRY(fwd_gemm<FE_GELU>(m_h16, m_ff1, p, s));
        p = base;
        p.N = d; p.K = ffn; p.w_row0 = l * d;
        ACB_TRY(fwd_gemm<FE_RESID>(m_f16, m_ff2, p, s));
    }
    ACB_TRY(ln(w->out_norm, w->out_norm + d));
    FwdGemmParams p = base;
    p.N = NV; p.w_row0 = 0;
    return fwd_gemm<FE_LOGITS>(m_h16, m_heads, p, s);
}
