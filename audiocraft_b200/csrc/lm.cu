// MusicGen LM decode step for H100 (sm_90a).
//
// One decode step = LMModel.forward on one token per row (audiocraft/models/lm.py:221-268) + CFG mix + sampling
// (lm.py:393-418) + the delay-pattern write-back (lm.py:553-562), replayed as ONE CUDA graph per step with every
// step-dependent quantity (position, tokens) resident on the device.
//
// The step is HBM-bound in bytes (all layer weights, fp16, 3.2 GB for medium, and the KV cache are read once per step at ~rows FLOP/B)
// and LATENCY-bound in time: 11 dependent kernels per layer, chained by plain stream-order edges of the graph.  Design consequences:
//   * weights stay in the reference's [out][in] fp16 layout; a CTA's 16 (or 32) x kslice slab is fetched with TMA bulk copies
//     issued before the CTA reads its first activation; a 16x32 block of W is the A operand of two m16n8k16 MMAs, the activations
//     (a few KB, L2 resident) are the B operand, so the tile is 16 output features x (8*NT) rows and nothing is wasted on padding
//     rows up to 128.
//   * every GEMM spreads its weight matrix over >= 2 CTAs per SM; small-N GEMMs split K across CTAs and the partial sums are reduced
//     (in a fixed order: bit-reproducible) by the consumer kernel, which is the residual add + LayerNorm, so that reduction costs no
//     extra pass.
//   * K/V go from the QKV GEMM epilogue straight into the cache; cross-attention K/V are computed once per generate() instead of
//     every step (the reference recomputes them, transformer.py:355-357).
//   * self attention: one CTA per (query row, head) streaming K and V through a cp.async ring (lm_attn2_kernel), for the decode
//     step and for prompt prefill alike.
#include "common.cuh"
#include "lm_math.cuh"
#include "tma.cuh"
#include "wgmma.cuh"
#include <cooperative_groups.h>
#include <cuda_fp8.h>
#include <math.h>
#include <new>
#include <vector>
#include <stdio.h>
#include <stdlib.h>

// Slot mode (acb_lm_begin_slots): per-slot device state, ACB_LM_SLOT_STRIDE ints per slot in buffers.slot_state.  The host
// writes a slot only at admission (lm_slot_admit_kernel); the step's sampler advances POS and sets STATUS to FINISHED.
// POS counts the sequence columns consumed; PREFIX is the slot's condition-prefix length, so column t runs at cache position
// PREFIX + t.
enum { ACB_SLOT_POS = 0, ACB_SLOT_STATUS = 1, ACB_SLOT_SEQ_LEN = 2, ACB_SLOT_TEXT_LEN = 3, ACB_SLOT_SEED_LO = 4,
       ACB_SLOT_SEED_HI = 5, ACB_SLOT_DONE = 6, ACB_SLOT_PREFIX = 7 };
enum { SLOT_INACTIVE = 0, SLOT_ACTIVE = 1, SLOT_FINISHED = 2 };

// ------------------------------------------------------------------------------------------------ helpers
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (UBLKCP in SASS). 16 B aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ float block_max(float v, float* red) {
    v = warp_max(v);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = lane < nw ? red[lane] : -INFINITY;
    return warp_max(t);
}

// ------------------------------------------------------------------------------------------------ embed + sin pos
// x[r] = sum_k emb_k[seq[b,k,pos]] + pos_scale * [cos(pos/f_i), sin(pos/f_i)]   (lm.py:244, transformer.py:70-89,701-705)
// The sin term only when sin_pos ('sin' and 'sin_rope'; a 'rope' model has its positions in the QKV epilogue alone).
// Shared by the per-generation kernel below and the slot-mode kernel (each row at its own position).
__device__ __forceinline__ void embed_row(const __half* __restrict__ emb, const float* __restrict__ inv_freq,
                                          const int64_t* __restrict__ seq, float* __restrict__ x, int r, int b, int pos,
                                          int d, int n_q, int card, int max_seq, float pos_scale, bool sin_pos, int seq_off) {
    __shared__ int tok[16];
    if (threadIdx.x < n_q) {
        long long t = seq[((size_t)b * n_q + threadIdx.x) * max_seq + pos - seq_off];
        tok[threadIdx.x] = (int)(t < 0 ? card : (t > card ? card : t));
    }
    __syncthreads();
    const int half_d = d >> 1;
    for (int i = threadIdx.x; i < d; i += 256) {   // d % 32 == 0: a warp is entirely inside or outside the row
        float v = 0.f;
        for (int k = 0; k < n_q; ++k) v += __half2float(emb[((size_t)k * (card + 1) + tok[k]) * d + i]);
        if (sin_pos) {
            const int j = i < half_d ? i : i - half_d;
            const float phase = (float)pos / inv_freq[j];
            v += pos_scale * (i < half_d ? cosf(phase) : sinf(phase));
        }
        x[(size_t)r * d + i] = v;
    }
}

// PF (prompt prefill): the grid's rows are (token, row) pairs r = tok * rows_real + row at positions P[0] + tok.
// seq_off: length of the condition prefix in front of the tokens; cache position pos reads sequence column pos - seq_off.
template <bool PF>
__global__ void __launch_bounds__(256) lm_embed_kernel(const __half* __restrict__ emb, const float* __restrict__ inv_freq,
                                                       const int64_t* __restrict__ seq, const int* __restrict__ P,
                                                       float* __restrict__ x, int d, int n_q, int card, int max_seq,
                                                       int batch, float pos_scale, int rows_real, bool sin_pos, int seq_off) {
    const int r = blockIdx.x, b = (PF ? r % rows_real : r) % batch, pos = P[0] + (PF ? r / rows_real : 0);
    embed_row(emb, inv_freq, seq, x, r, b, pos, d, n_q, card, max_seq, pos_scale, sin_pos, seq_off);
}

// Slot mode (continuous batching): row r belongs to slot r % slots (cond rows [0, slots), null rows [slots, 2 slots)) and
// reads that slot's sequence column at the slot's own position; the sin term is at cache position prefix + column, as
// lm_embed_kernel's seq_off has it.  An inactive slot embeds a finite, unused row.
__global__ void __launch_bounds__(256) lm_embed_slot_kernel(const __half* __restrict__ emb, const float* __restrict__ inv_freq,
                                                            const int64_t* __restrict__ seq, const int* __restrict__ slot_state,
                                                            float* __restrict__ x, int d, int n_q, int card, int max_seq,
                                                            int slots, float pos_scale, bool sin_pos) {
    const int r = blockIdx.x, b = r % slots;
    const int* st = slot_state + b * ACB_LM_SLOT_STRIDE;
    const int prefix = st[ACB_SLOT_PREFIX];
    embed_row(emb, inv_freq, seq, x, r, b, prefix + st[ACB_SLOT_POS], d, n_q, card, max_seq, pos_scale, sin_pos, prefix);
}

// Condition-prefix prefill (the `prepend` fuser, conditioners.py:1703-1763): the grid's rows are (position, row) pairs
// r = p * rows_real + row at cache positions P[0] + p, and x[r] = prefix[row][P[0] + p] (rounded to fp16 like the reference's
// autocast output_proj) + the sin term.  Each row has its own prefix: cond and null rows differ.
__global__ void __launch_bounds__(256) lm_embed_prefix_kernel(const float* __restrict__ prefix, const float* __restrict__ inv_freq,
                                                              const int* __restrict__ P, float* __restrict__ x, int d,
                                                              int prefix_len, float pos_scale, int rows_real, bool sin_pos) {
    const int r = blockIdx.x, row = r % rows_real, pos = P[0] + r / rows_real;
    const float* src = prefix + ((size_t)row * prefix_len + pos) * d;
    const int half_d = d >> 1;
    for (int i = threadIdx.x; i < d; i += 256) {
        float v = half_round(src[i]);
        if (sin_pos) {
            const int j = i < half_d ? i : i - half_d;
            const float phase = (float)pos / inv_freq[j];
            v += pos_scale * (i < half_d ? cosf(phase) : sinf(phase));
        }
        x[(size_t)r * d + i] = v;
    }
}

// ------------------------------------------------------------------------------------------------ residual + LN
// x[r] += sum_s part[s][r] (fixed order), then h16[r] = LayerNorm(x[r]) * gamma + beta  (eps 1e-5, fp32 statistics).
// One CTA per row, ONE float4 per thread (d <= 2048): no per-thread loops, so the kernel is ~300 instructions -- at this
// time scale cold instruction fetch is a first-order cost (a 4-float4-per-thread version was over 1 000 instructions).
constexpr int LN_THREADS = 512;
__global__ void __launch_bounds__(LN_THREADS) lm_ln_kernel(float* __restrict__ x, const float* __restrict__ part, int nsplit,
                                                           size_t split_stride, const float* __restrict__ gamma,
                                                           const float* __restrict__ beta, __half* __restrict__ out, int d) {
    __shared__ float red[2][32];
    const int r = blockIdx.x, i = threadIdx.x;
    const bool live = i < (d >> 2);
    float4 gm = make_float4(0.f, 0.f, 0.f, 0.f), bt = gm;
    if (live) { gm = reinterpret_cast<const float4*>(gamma)[i]; bt = reinterpret_cast<const float4*>(beta)[i]; }
    float4* xr = reinterpret_cast<float4*>(x + (size_t)r * d);
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (live) {
        a = xr[i];
        float4 pt[ACB_LM_MAX_SPLIT];
#pragma unroll
        for (int sp = 0; sp < ACB_LM_MAX_SPLIT; ++sp)   // independent loads, all in flight together
            pt[sp] = sp < nsplit ? reinterpret_cast<const float4*>(part + sp * split_stride + (size_t)r * d)[i]
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int sp = 0; sp < ACB_LM_MAX_SPLIT; ++sp) {  // fixed summation order
            a.x += pt[sp].x; a.y += pt[sp].y; a.z += pt[sp].z; a.w += pt[sp].w;
        }
        if (nsplit) xr[i] = a;
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

// ------------------------------------------------------------------------------------------------ skinny GEMM
// _PF: prompt prefill, rows are (token, row) pairs; _ROPE: q and k rotated (rotary positions) before they are stored
enum { EPI_PARTIAL = 0, EPI_QKV = 1, EPI_GELU = 2, EPI_F32 = 3, EPI_CROSSKV = 4, EPI_QKV_PF = 5, EPI_QKV_ROPE = 6, EPI_QKV_PF_ROPE = 7 };

// The rotary fields live in padding and in a field the QKV epilogues do not use, so the struct keeps its size and offsets:
// ptxas schedules every instance by the parameter layout, and 16 more bytes made the MusicGen-medium decode GEMM pass 2 %
// slower (2.68 vs 2.62 ms, H100 80GB HBM3 at a 400 W limit).
struct GemmParams {
    const __half* W;  // [N][K] fp16, reference layout
    const __half* X;  // [8*NT][K] fp16, rows >= `rows` are zero
    int N, K, rows, kslice;                            // kslice: K elements per CTA (grid.y slices)
    float* out_f32; int ld_out;                        // PARTIAL / F32
    float pos_scale;                                   // QKV_ROPE / QKV_PF_ROPE: positional_scale
    size_t split_stride;                               // PARTIAL
    union {
        __half* out_f16;                               // GELU
        const float* rope_freq;                        // QKV_ROPE / QKV_PF_ROPE: [32] RotaryEmbedding.frequencies
    };
    float* q32; __half* kc; __half* vc; int d, H, cache_len; const int* pos;  // QKV / CROSSKV
    int text_len, row0;                                                      // CROSSKV
    int rows_real;                                                           // QKV_PF: rows of the generation (GEMM row = tok * rows_real + row)
    int row_stride;   // QKV_PF: row `row` of the generation is cache row row * row_stride of kc / vc (slots in an admission, else 1)
};
static_assert(sizeof(GemmParams) == 128, "GemmParams layout");

// RotaryEmbedding.rotate_qk (modules/rope.py:84-125) on one fp16 element of q / k at position pos: the head dim is 32 complex
// pairs (2i, 2i+1), rotated by pos * max_period^(-2i/64) in fp32 and blended with `pos_scale`; `other` is the pair partner.
// Out of line: sincosf is large and rotary positions are an option, not the released models' default.
__device__ __noinline__ float rope_rotate(const float* rope_freq, float pos_scale, float vh, float other, int dd, int pos) {
    const bool even = (dd & 1) == 0;
    const float re = even ? vh : other, im = even ? other : vh;
    const float ang = (float)pos * rope_freq[dd >> 1];
    float sn, cs;
    sincosf(ang, &sn, &cs);
    const float rr = cs * pos_scale + (1.f - pos_scale), ri = sn * pos_scale;
    return even ? re * rr - im * ri : re * ri + im * rr;
}

// FP8 weights (acb_lm_config.weight_dtype = 1): two e4m3 codes -> two fp16 values, exactly (every e4m3 value is an fp16
// value); the upper byte becomes the upper half.
__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint32_t two_codes) {
    uint32_t r;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"((uint16_t)two_codes));
    return r;
}
// 8 codes (k .. k + 7, k at the lowest byte) -> the 8 fp16 values an fp16 slab holds in one uint4
__device__ __forceinline__ uint4 e4m3x8_to_f16x8(uint2 c) {
    return make_uint4(e4m3x2_to_f16x2(c.x), e4m3x2_to_f16x2(c.x >> 16), e4m3x2_to_f16x2(c.y), e4m3x2_to_f16x2(c.y >> 16));
}

// Bytes per staged weight row: fp16 as lm_gemm_kernel computes it (+64 for conflict-free LDS.128), e4m3 for lm_gemm_fp8_kernel.
// e4m3: rows 32 bytes apart modulo 128, so the 4 rows one half-warp's LDS.64 touch lie in 4 different 8-bank groups.
__host__ __device__ __forceinline__ int gemm_pitch(int kslice, bool w8) {
    return w8 ? (kslice + 127) / 128 * 128 + 32 : kslice * 2 + 64;
}

// CTA = 4 warps, tile = 16 output features x kslice of K.  The CTA's 16 x kslice weight slab is fetched by ONE thread
// with 16 TMA bulk copies (one per W row, padded pitch => conflict-free fragment reads), issued before the first activation
// read so that the weight bytes are in flight while the activations load.
// FT2 = feature tiles of 16 per CTA.  FT2 = 2 (opt-in per GEMM, see pick_ft2) halves the number of CTAs and therefore
// the activation traffic out of L2: every CTA re-reads the whole 16 x K activation block, as many bytes as the weights.
template <int NT, int EPI, int FT2 = 1>
__global__ void __launch_bounds__(128) lm_gemm_kernel(GemmParams p) {
    constexpr int U = NT <= 2 ? 4 : (NT <= 4 ? 2 : 1);   // k-blocks per batch of activation loads
    constexpr int RP = 8 * NT + 1;
    constexpr int FB = 16 * FT2;                     // output features per CTA
    constexpr bool ROPE = EPI == EPI_QKV_ROPE || EPI == EPI_QKV_PF_ROPE, PF = EPI == EPI_QKV_PF || EPI == EPI_QKV_PF_ROPE;
    constexpr bool QKV = EPI == EPI_QKV || PF || ROPE;
    extern __shared__ __align__(128) unsigned char gsm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c4 = lane & 3;
    const int f0 = blockIdx.x * FB;
    const int k0 = blockIdx.y * p.kslice;
    const int ks = min(p.kslice, p.K - k0);          // elements of K this CTA reduces over
    const int pitch = p.kslice * 2 + 64;             // bytes per staged W row (+64: conflict-free LDS.128)
    uint64_t* bar = reinterpret_cast<uint64_t*>(gsm + FB * pitch);
    float* red = reinterpret_cast<float*>(gsm + FB * pitch + 16);   // [4][FB][RP]

    if (tid == 0) mbar_init(bar, 1);
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(bar, (uint32_t)FB * (uint32_t)ks * 2u);
#pragma unroll 1
        for (int r = 0; r < FB; ++r)
            bulk_g2s(gsm + r * pitch, p.W + (size_t)(f0 + r) * p.K + k0, (uint32_t)ks * 2u, bar);
    }
    int cache_pos = 0;
    if (QKV) cache_pos = p.pos[0];   // requested now, consumed in the epilogue: off the critical path

    float c[FT2][NT][4];
#pragma unroll
    for (int ft = 0; ft < FT2; ++ft)
#pragma unroll
        for (int j = 0; j < NT; ++j) c[ft][j][0] = c[ft][j][1] = c[ft][j][2] = c[ft][j][3] = 0.f;

    const int nkb = ks >> 5;
    const int kbw = (nkb + 3) >> 2;
    const int kb0 = min(nkb, warp * kbw), kb1 = min(nkb, kb0 + kbw);
    const __half* xr = p.X + (size_t)g * p.K + k0 + 8 * c4;
    const unsigned char* wr0 = gsm + g * pitch + 16 * c4;
    const unsigned char* wr1 = wr0 + 8 * pitch;

    bool w_ready = false;
    for (int kb = kb0; kb < kb1; kb += U) {
        uint4 xv[U][NT];
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
            for (int j = 0; j < NT; ++j)
                xv[u][j] = (kb + u < kb1) ? *reinterpret_cast<const uint4*>(xr + (size_t)(8 * j) * p.K + (size_t)(kb + u) * 32)
                                          : make_uint4(0, 0, 0, 0);
        if (!w_ready) { mbar_wait(bar, 0); w_ready = true; }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (kb + u < kb1) {
#pragma unroll
                for (int ft = 0; ft < FT2; ++ft) {
                    const uint4 wa = *reinterpret_cast<const uint4*>(wr0 + ft * 16 * pitch + (kb + u) * 64);
                    const uint4 wb = *reinterpret_cast<const uint4*>(wr1 + ft * 16 * pitch + (kb + u) * 64);
#pragma unroll
                    for (int j = 0; j < NT; ++j) {
                        mma16816(c[ft][j], wa.x, wb.x, wa.y, wb.y, xv[u][j].x, xv[u][j].y);
                        mma16816(c[ft][j], wa.z, wb.z, wa.w, wb.w, xv[u][j].z, xv[u][j].w);
                    }
                }
            }
        }
    }
    if (!w_ready) mbar_wait(bar, 0);   // never leave with a bulk copy in flight
    // cross-warp (split-K inside the CTA) reduction in a fixed order
#pragma unroll
    for (int ft = 0; ft < FT2; ++ft)
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            float* r0 = red + (warp * FB + ft * 16 + g) * RP + 8 * j + 2 * c4;
            r0[0] = c[ft][j][0];
            r0[1] = c[ft][j][1];
            r0[8 * RP] = c[ft][j][2];
            r0[8 * RP + 1] = c[ft][j][3];
        }
    __syncthreads();
    for (int idx = tid; idx < FB * 8 * NT; idx += 128) {
        const int row = idx / FB, feat = idx % FB;
        if (row >= p.rows) continue;
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) v += red[(w * FB + feat) * RP + row];
        const int n = f0 + feat;
        if (EPI == EPI_PARTIAL) {
            p.out_f32[blockIdx.y * p.split_stride + (size_t)row * p.ld_out + n] = v;
        } else if (EPI == EPI_F32) {
            p.out_f32[(size_t)row * p.ld_out + n] = v;
        } else if (EPI == EPI_GELU) {
            p.out_f16[(size_t)row * p.ld_out + n] = __float2half_rn(gelu_erf(half_round(v)));
        } else if (QKV) {   // q | k | v blocks of d features each (no integer division: cold code costs here)
            // prefill: row = tk * rows_real + rr -> cache row rr * row_stride, position cache_pos + tk
            const int which = n >= 2 * p.d ? 2 : (n >= p.d ? 1 : 0), nn = n - which * p.d;
            const int tk = PF ? row / p.rows_real : 0, rr = PF ? (row - tk * p.rows_real) * p.row_stride : row;
            if (ROPE && which < 2) {   // the pair partner is feature n ^ 1 of the same CTA (f0 % 16 == 0), same warp order
                float other = 0.f;
#pragma unroll
                for (int w = 0; w < 4; ++w) other += red[(w * FB + (feat ^ 1)) * RP + row];
                v = rope_rotate(p.rope_freq, p.pos_scale, half_round(v), half_round(other), nn & 63, cache_pos + tk);
            }
            if (which == 0) {
                p.q32[(size_t)row * p.d + nn] = v;
            } else {
                __half* cache = which == 2 ? p.vc : p.kc;
                cache[(((size_t)rr * p.H + (nn >> 6)) * p.cache_len + cache_pos + tk) * 64 + (nn & 63)] = __float2half_rn(v);
            }
        } else {  // EPI_CROSSKV: GEMM rows are (row, text position) pairs
            const int R = p.row0 + row, r = R / p.text_len, tc = R % p.text_len;
            const int which = n / p.d, nn = n % p.d, h = nn >> 6, dd = nn & 63;
            __half* cache = which ? p.vc : p.kc;
            cache[(((size_t)r * p.H + h) * p.cache_len + tc) * 64 + dd] = __float2half_rn(v);
        }
    }
}

// lm_gemm_kernel on FP8 weights (acb_lm_config.weight_dtype = 1), a kernel of its own so that the fp16 instances keep their
// code and their parameter layout: the same tiles, split, FT2 and epilogues.  The slab is e4m3 codes (p.W points at bytes);
// each lane reads 8 codes where the fp16 slab gives it 8 halves, so the k order against the activations is the fp16 one, and
// unpacks them exactly to fp16 for the same MMAs.  wscale[n] (the row's fp32 scale) multiplies output n's fixed-order sum
// once, before the epilogue does anything else with it (an EPI_PARTIAL slice is scaled before it is stored).
// (128, 4): without the occupancy target ptxas spilled 8 bytes in <2, EPI_QKV, 2>; with it no instance spills.
template <int NT, int EPI, int FT2 = 1>
__global__ void __launch_bounds__(128, 4) lm_gemm_fp8_kernel(GemmParams p, const float* __restrict__ wscale) {
    constexpr int U = NT <= 2 ? 4 : (NT <= 4 ? 2 : 1);   // k-blocks per batch of activation loads
    constexpr int RP = 8 * NT + 1;
    constexpr int FB = 16 * FT2;                     // output features per CTA
    constexpr bool ROPE = EPI == EPI_QKV_ROPE || EPI == EPI_QKV_PF_ROPE, PF = EPI == EPI_QKV_PF || EPI == EPI_QKV_PF_ROPE;
    constexpr bool QKV = EPI == EPI_QKV || PF || ROPE;
    extern __shared__ __align__(128) unsigned char gsm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c4 = lane & 3;
    const int f0 = blockIdx.x * FB;
    const int k0 = blockIdx.y * p.kslice;
    const int ks = min(p.kslice, p.K - k0);          // elements of K this CTA reduces over
    const int pitch = gemm_pitch(p.kslice, true);    // bytes per staged W row
    uint64_t* bar = reinterpret_cast<uint64_t*>(gsm + FB * pitch);
    float* red = reinterpret_cast<float*>(gsm + FB * pitch + 16);   // [4][FB][RP]

    if (tid == 0) mbar_init(bar, 1);
    __syncthreads();
    if (tid == 0) {
        const uint8_t* wc = reinterpret_cast<const uint8_t*>(p.W);   // codes: one byte per weight
        mbar_expect_tx(bar, (uint32_t)FB * (uint32_t)ks);
#pragma unroll 1
        for (int r = 0; r < FB; ++r) bulk_g2s(gsm + r * pitch, wc + (size_t)(f0 + r) * p.K + k0, (uint32_t)ks, bar);
    }
    int cache_pos = 0;
    if (QKV) cache_pos = p.pos[0];   // requested now, consumed in the epilogue: off the critical path

    float c[FT2][NT][4];
#pragma unroll
    for (int ft = 0; ft < FT2; ++ft)
#pragma unroll
        for (int j = 0; j < NT; ++j) c[ft][j][0] = c[ft][j][1] = c[ft][j][2] = c[ft][j][3] = 0.f;

    const int nkb = ks >> 5;
    const int kbw = (nkb + 3) >> 2;
    const int kb0 = min(nkb, warp * kbw), kb1 = min(nkb, kb0 + kbw);
    const __half* xr = p.X + (size_t)g * p.K + k0 + 8 * c4;
    const unsigned char* wr0 = gsm + g * pitch + 8 * c4;
    const unsigned char* wr1 = wr0 + 8 * pitch;

    bool w_ready = false;
    for (int kb = kb0; kb < kb1; kb += U) {
        uint4 xv[U][NT];
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
            for (int j = 0; j < NT; ++j)
                xv[u][j] = (kb + u < kb1) ? *reinterpret_cast<const uint4*>(xr + (size_t)(8 * j) * p.K + (size_t)(kb + u) * 32)
                                          : make_uint4(0, 0, 0, 0);
        if (!w_ready) { mbar_wait(bar, 0); w_ready = true; }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (kb + u < kb1) {
#pragma unroll
                for (int ft = 0; ft < FT2; ++ft) {
                    const uint4 wa = e4m3x8_to_f16x8(*reinterpret_cast<const uint2*>(wr0 + ft * 16 * pitch + (kb + u) * 32));
                    const uint4 wb = e4m3x8_to_f16x8(*reinterpret_cast<const uint2*>(wr1 + ft * 16 * pitch + (kb + u) * 32));
#pragma unroll
                    for (int j = 0; j < NT; ++j) {
                        mma16816(c[ft][j], wa.x, wb.x, wa.y, wb.y, xv[u][j].x, xv[u][j].y);
                        mma16816(c[ft][j], wa.z, wb.z, wa.w, wb.w, xv[u][j].z, xv[u][j].w);
                    }
                }
            }
        }
    }
    if (!w_ready) mbar_wait(bar, 0);   // never leave with a bulk copy in flight
    // cross-warp (split-K inside the CTA) reduction in a fixed order
#pragma unroll
    for (int ft = 0; ft < FT2; ++ft)
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            float* r0 = red + (warp * FB + ft * 16 + g) * RP + 8 * j + 2 * c4;
            r0[0] = c[ft][j][0];
            r0[1] = c[ft][j][1];
            r0[8 * RP] = c[ft][j][2];
            r0[8 * RP + 1] = c[ft][j][3];
        }
    __syncthreads();
    for (int idx = tid; idx < FB * 8 * NT; idx += 128) {
        const int row = idx / FB, feat = idx % FB;
        if (row >= p.rows) continue;
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) v += red[(w * FB + feat) * RP + row];
        const int n = f0 + feat;
        v *= wscale[n];   // the row scale, once, on the fixed-order sum
        if (EPI == EPI_PARTIAL) {
            p.out_f32[blockIdx.y * p.split_stride + (size_t)row * p.ld_out + n] = v;
        } else if (EPI == EPI_F32) {
            p.out_f32[(size_t)row * p.ld_out + n] = v;
        } else if (EPI == EPI_GELU) {
            p.out_f16[(size_t)row * p.ld_out + n] = __float2half_rn(gelu_erf(half_round(v)));
        } else if (QKV) {   // q | k | v blocks of d features each (no integer division: cold code costs here)
            // prefill: row = tk * rows_real + rr -> cache row rr * row_stride, position cache_pos + tk
            const int which = n >= 2 * p.d ? 2 : (n >= p.d ? 1 : 0), nn = n - which * p.d;
            const int tk = PF ? row / p.rows_real : 0, rr = PF ? (row - tk * p.rows_real) * p.row_stride : row;
            if (ROPE && which < 2) {   // the pair partner is feature n ^ 1 of the same CTA (f0 % 16 == 0), same warp order
                float other = 0.f;
#pragma unroll
                for (int w = 0; w < 4; ++w) other += red[(w * FB + (feat ^ 1)) * RP + row];
                other *= wscale[n ^ 1];
                v = rope_rotate(p.rope_freq, p.pos_scale, half_round(v), half_round(other), nn & 63, cache_pos + tk);
            }
            if (which == 0) {
                p.q32[(size_t)row * p.d + nn] = v;
            } else {
                __half* cache = which == 2 ? p.vc : p.kc;
                cache[(((size_t)rr * p.H + (nn >> 6)) * p.cache_len + cache_pos + tk) * 64 + (nn & 63)] = __float2half_rn(v);
            }
        } else {  // EPI_CROSSKV: GEMM rows are (row, text position) pairs
            const int R = p.row0 + row, r = R / p.text_len, tc = R % p.text_len;
            const int which = n / p.d, nn = n % p.d, h = nn >> 6, dd = nn & 63;
            __half* cache = which ? p.vc : p.kc;
            cache[(((size_t)r * p.H + h) * p.cache_len + tc) * 64 + dd] = __float2half_rn(v);
        }
    }
}

// ------------------------------------------------------------------------------------------------ wide GEMM (65-256 rows)
// The decode GEMM for rows > 64, where lm_gemm_kernel's mma.sync tile (8 * NT <= 64 rows in registers) cannot grow.  Swap-AB
// on wgmma: the output tile is 64 features x all NPAD rows, D = W[64 x k] . X[NPAD x k]^T with the weight slab as the A
// operand and the activations as the B operand, both K-major in the 128-byte swizzle that tiled TMA writes.  One CTA covers
// every row of its features, so each weight byte is read from HBM once per step whatever the batch.  The weights stay in the
// reference's [N][K] layout: one 2-D tensor map per stacked matrix ([L * N][K]), the layer is a row offset.
// NPAD is 128 (rows 65-128) or 256 (rows 129-256): the padded rows cost MMA issue slots and L2 reads of zero-filled
// activations, not HBM bytes, and two widths keep the instance count (and the build) small.
// K is cut into 64-element chunks streamed through an mbarrier ring.  The K split (grid.y) depends only on (N, K, SM count):
// EPI_PARTIAL writes one `part` slot per slice, the other epilogues split K over a thread-block cluster of grid.y CTAs and
// add the slices' tiles in rank order through distributed shared memory.  An item's sums are therefore the same in every
// batch of this range.
constexpr int WIDE_KC = 64;   // K elements per chunk: one 128-byte swizzle row
static_assert(WIDE_KC == TMA_BOX_K, "the tensor maps (encode_map) deliver one chunk per box");
template <int NPAD, int W_ELEM_BYTES = 2>
struct WideCfg {
    static constexpr int W_BYTES = 64 * WIDE_KC * W_ELEM_BYTES;
    static constexpr int STAGE = W_BYTES + NPAD * WIDE_KC * 2;
    static constexpr int STAGES = NPAD <= 128 ? 6 : 5;
    static constexpr int LDS = 68;   // pitch (floats) of the [NPAD][64] fp32 staging tile: conflict-free fragment stores
    static constexpr int SMEM = STAGES * STAGE + 1024 + 64;   // ring (1024-aligned) + barriers
    static_assert(NPAD * LDS * 4 <= STAGES * STAGE, "the staging tile reuses the ring");
};

// EPI is EPI_PARTIAL, EPI_QKV, EPI_QKV_ROPE, EPI_GELU or EPI_F32.  Prefill passes above 64 rows carry one position per row,
// so their QKV epilogue is the decode one (token 0 of the pass at position pos).
// W8 (FP8 weights): the weight chunk is 64 rows x 64 e4m3 codes, staged by a uint8 map with the 64-byte swizzle (16-byte
// unit c of row r at unit c ^ ((r >> 1) & 3)), so the 8 rows of one LDS.U16 fall in 8 different 4-bank groups.  Each warp
// unpacks its 16 rows into the A fragment in registers (exact fp16), the MMAs take A from registers and the activations from
// the same swizzled stage as in fp16, and wscale[n] multiplies output n's sum after the cluster's fixed-order reduction.
template <int NPAD, int EPI, bool W8>
__device__ __forceinline__ void wide_body(const CUtensorMap& wmap, const CUtensorMap& xmap, const GemmParams& p, int w_row0,
                                          const float* __restrict__ wscale) {
    using Cfg = WideCfg<NPAD, W8 ? 1 : 2>;
    constexpr bool ROPE = EPI == EPI_QKV_ROPE, QKV = EPI == EPI_QKV || ROPE;
    extern __shared__ unsigned char wsm_raw[];
    unsigned char* wsm = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(wsm_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(wsm + Cfg::STAGES * Cfg::STAGE);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int f0 = blockIdx.x * 64, k0 = blockIdx.y * p.kslice;
    const int nch = (min(p.kslice, p.K - k0) + WIDE_KC - 1) / WIDE_KC;   // K past the end is zero-filled by TMA

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < Cfg::STAGES; ++s) mbar_init(&full[s], 1);
    }
    __syncthreads();
    auto load = [&](int c) {
        const int s = c % Cfg::STAGES;
        unsigned char* st = wsm + s * Cfg::STAGE;
        mbar_expect_tx(&full[s], (uint32_t)Cfg::STAGE);
        tma_load_2d(st, &wmap, k0 + c * WIDE_KC, w_row0 + f0, &full[s]);
        tma_load_2d(st + Cfg::W_BYTES, &xmap, k0 + c * WIDE_KC, 0, &full[s]);   // rows >= p.rows are zero-filled
    };
    if (tid == 0)
        for (int c = 0; c < min(nch, Cfg::STAGES); ++c) load(c);
    int cache_pos = 0;
    if (QKV) cache_pos = p.pos[0];

    float acc[NPAD / 2];
#pragma unroll
    for (int i = 0; i < NPAD / 2; ++i) acc[i] = 0.f;
    for (int c = 0; c < nch; ++c) {
        const int s = c % Cfg::STAGES;
        mbar_wait(&full[s], (uint32_t)(c / Cfg::STAGES) & 1u);
        const uint32_t a = smem_u32(wsm + s * Cfg::STAGE), b = a + Cfg::W_BYTES;
        if constexpr (W8) {
            // lane (g, c4) of warp w: codes k = 16 kk + 2 c4 (+1) and + 8 of rows 16 w + g and 16 w + g + 8
            const int g = lane >> 2, c4 = lane & 3, r0 = 16 * warp + g, r1 = r0 + 8;
            const unsigned char* st = wsm + s * Cfg::STAGE;
            uint32_t af[WIDE_KC / 16][4];
#pragma unroll
            for (int kk = 0; kk < WIDE_KC / 16; ++kk) {
                const int o0 = r0 * 64 + 16 * (kk ^ ((r0 >> 1) & 3)) + 2 * c4, o1 = r1 * 64 + 16 * (kk ^ ((r1 >> 1) & 3)) + 2 * c4;
                af[kk][0] = e4m3x2_to_f16x2(*reinterpret_cast<const uint16_t*>(st + o0));
                af[kk][1] = e4m3x2_to_f16x2(*reinterpret_cast<const uint16_t*>(st + o1));
                af[kk][2] = e4m3x2_to_f16x2(*reinterpret_cast<const uint16_t*>(st + o0 + 8));
                af[kk][3] = e4m3x2_to_f16x2(*reinterpret_cast<const uint16_t*>(st + o1 + 8));
            }
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < WIDE_KC / 16; ++kk) wgmma_f16_ra<NPAD>(acc, af[kk], wgmma_desc_sw128(b + 32 * kk), 1u);
        } else {
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < WIDE_KC / 16; ++kk)   // a 16-element K step advances the start address by 32 bytes
                wgmma_f16<NPAD>(acc, wgmma_desc_sw128(a + 32 * kk), wgmma_desc_sw128(b + 32 * kk), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (c + Cfg::STAGES < nch) {   // every warp is done with stage s: refill it
            __syncthreads();
            if (tid == 0) load(c + Cfg::STAGES);
        }
    }
    __syncthreads();   // the ring is idle: it becomes the staging tile [row][feature]
    float* tile = reinterpret_cast<float*>(wsm);
#pragma unroll
    for (int j = 0; j < NPAD / 8; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i)
            tile[(8 * j + 2 * (lane & 3) + (i & 1)) * Cfg::LDS + 16 * warp + (lane >> 2) + 8 * (i >> 1)] = acc[4 * j + i];

    namespace cg = cooperative_groups;
    const int cs = EPI == EPI_PARTIAL ? 1 : (int)gridDim.y;   // CTAs of the cluster that share this tile's K
    const float* src[4] = {tile, tile, tile, tile};
    int rank = 0;
    if (cs > 1) {
        cg::cluster_group cluster = cg::this_cluster();
        cluster.sync();
        rank = (int)cluster.block_rank();
#pragma unroll
        for (int r = 0; r < 4; ++r)
            if (r < cs) src[r] = cluster.map_shared_rank(tile, r);
    } else {
        __syncthreads();
    }
    const int per = (p.rows + cs - 1) / cs, r0 = rank * per, r1 = min(p.rows, r0 + per);   // this CTA's output rows
    for (int idx = tid; idx < (r1 - r0) * 64; idx += 128) {
        const int row = r0 + (idx >> 6), feat = idx & 63, n = f0 + feat;
        float v = 0.f;
#pragma unroll
        for (int r = 0; r < 4; ++r)   // fixed order: slice 0 first
            if (r < cs) v += src[r][row * Cfg::LDS + feat];
        if constexpr (W8) v *= wscale[n];
        if (EPI == EPI_PARTIAL) {
            p.out_f32[blockIdx.y * p.split_stride + (size_t)row * p.ld_out + n] = v;
        } else if (EPI == EPI_F32) {
            p.out_f32[(size_t)row * p.ld_out + n] = v;
        } else if (EPI == EPI_GELU) {
            p.out_f16[(size_t)row * p.ld_out + n] = __float2half_rn(gelu_erf(half_round(v)));
        } else if (QKV) {
            const int which = n >= 2 * p.d ? 2 : (n >= p.d ? 1 : 0), nn = n - which * p.d;
            if (ROPE && which < 2) {   // the pair partner n ^ 1 is in the same 64-feature tile
                float other = 0.f;
#pragma unroll
                for (int r = 0; r < 4; ++r)
                    if (r < cs) other += src[r][row * Cfg::LDS + (feat ^ 1)];
                if constexpr (W8) other *= wscale[n ^ 1];
                v = rope_rotate(p.rope_freq, p.pos_scale, half_round(v), half_round(other), nn & 63, cache_pos);
            }
            if (which == 0) {
                p.q32[(size_t)row * p.d + nn] = v;
            } else {
                __half* cache = which == 2 ? p.vc : p.kc;
                cache[(((size_t)row * p.H + (nn >> 6)) * p.cache_len + cache_pos) * 64 + (nn & 63)] = __float2half_rn(v);
            }
        }
    }
    if (cs > 1) cg::this_cluster().sync();   // the other CTAs read this CTA's tile until here
}

template <int NPAD, int EPI>
__global__ void __launch_bounds__(128, 1) lm_gemm_wide_kernel(const __grid_constant__ CUtensorMap wmap,
                                                              const __grid_constant__ CUtensorMap xmap, GemmParams p, int w_row0) {
    wide_body<NPAD, EPI, false>(wmap, xmap, p, w_row0, nullptr);
}

template <int NPAD, int EPI>
__global__ void __launch_bounds__(128, 1) lm_gemm_wide_fp8_kernel(const __grid_constant__ CUtensorMap wmap,
                                                                  const __grid_constant__ CUtensorMap xmap, GemmParams p,
                                                                  int w_row0, const float* __restrict__ wscale) {
    wide_body<NPAD, EPI, true>(wmap, xmap, p, w_row0, wscale);
}

// Which cache position a row of a decode step or of a prompt pass appends at (and attends up to), shared by the fp16 and FP8
// QKV and attention kernels.
// Decode step (slot mode): row `row` belongs to slot row % slots and is at its cache position prefix + column.  Only the rows
// of an ACTIVE slot append or attend, and only they look their page up in `table` (a paged cache; null for a contiguous
// one or where the caller stages the whole table row): a slot not decoding owns no page.
struct SlotRow { int pos, page; bool live; };
__device__ __forceinline__ SlotRow slot_row(const int* __restrict__ slot_state, int slots, int row, const int* __restrict__ table,
                                            int pages_per_row) {
    const int* slot = slot_state + (row % slots) * ACB_LM_SLOT_STRIDE;
    SlotRow r;
    r.pos = slot[ACB_SLOT_PREFIX] + slot[ACB_SLOT_POS];
    r.live = slot[ACB_SLOT_STATUS] == SLOT_ACTIVE;
    r.page = r.live && table ? table[row * pages_per_row + r.pos / ACB_LM_KV_PAGE] : 0;
    return r;
}

// Prompt pass in a paged session (acb_lm_admit_prompt): GEMM row `row` is position P[0] + row / rows_real of generation row
// j = row % rows_real, whose page-table row is r0 + j * row_stride.
struct PassRow { int pos, trow; };
__device__ __forceinline__ PassRow pass_row(const int* __restrict__ P, int row, int rows_real, int r0, int row_stride) {
    const int tk = row / rows_real;
    return {P[0] + tk, r0 + (row - tk * rows_real) * row_stride};
}

// Slot mode's QKV epilogue and the paged prompt pass's, as kernels of their own: the QKV GEMM runs with the plain fp32
// epilogue (EPI_F32, the same sums as EPI_QKV / EPI_QKV_ROPE / EPI_QKV_PF*) into qkv [rows][3d], and these kernels do what
// those epilogues do at each row's own cache position pos: q to q32 (fp32), k and v to the cache (fp16), q and k rotated
// first under rotary positions, so q, k and v are bit-identical to the epilogues'.
// One row: k and v go to the cache only when `live`, each head's vector at ((x * H + head) * len + at) * 64, with x = row,
// len = cache_len, at = pos in a contiguous cache [rows][H][cache_len][64], and x = the page holding pos, len =
// ACB_LM_KV_PAGE, at = pos % ACB_LM_KV_PAGE in a page pool [n_pages][H][ACB_LM_KV_PAGE][64].
__device__ __forceinline__ void qkv_f16_row(const float* __restrict__ src, float* __restrict__ q32, __half* __restrict__ kc,
                                            __half* __restrict__ vc, int d, int H, const float* __restrict__ rope_freq,
                                            float pos_scale, bool rope, int row, int pos, int x, int len, int at, bool live) {
    for (int n = threadIdx.x; n < 3 * d; n += 256) {
        const int which = n >= 2 * d ? 2 : (n >= d ? 1 : 0), nn = n - which * d;
        float v = src[n];
        if (rope && which < 2) v = rope_rotate(rope_freq, pos_scale, half_round(v), half_round(src[n ^ 1]), nn & 63, pos);
        if (which == 0) {
            q32[(size_t)row * d + nn] = v;
        } else if (live) {
            __half* cache = which == 2 ? vc : kc;
            cache[(((size_t)x * H + (nn >> 6)) * len + at) * 64 + (nn & 63)] = __float2half_rn(v);
        }
    }
}

__global__ void __launch_bounds__(256) lm_qkv_slot_kernel(const float* __restrict__ qkv, const int* __restrict__ slot_state,
                                                          float* __restrict__ q32, __half* __restrict__ kc, __half* __restrict__ vc,
                                                          int d, int H, int cache_len, int slots, const float* __restrict__ rope_freq,
                                                          float pos_scale, bool rope) {
    const int row = blockIdx.x;
    const SlotRow r = slot_row(slot_state, slots, row, nullptr, 0);
    qkv_f16_row(qkv + (size_t)row * 3 * d, q32, kc, vc, d, H, rope_freq, pos_scale, rope, row, r.pos, row, cache_len, r.pos,
                r.live);
}

// Paged session (acb_lm_begin_slots_paged): kc / vc are the layer's page pool.
__global__ void __launch_bounds__(256) lm_qkv_slot_paged_kernel(const float* __restrict__ qkv, const int* __restrict__ slot_state,
                                                                float* __restrict__ q32, __half* __restrict__ kc,
                                                                __half* __restrict__ vc, int d, int H, int slots,
                                                                const float* __restrict__ rope_freq, float pos_scale, bool rope,
                                                                const int* __restrict__ table, int pages_per_row) {
    const int row = blockIdx.x;
    const SlotRow r = slot_row(slot_state, slots, row, table, pages_per_row);
    qkv_f16_row(qkv + (size_t)row * 3 * d, q32, kc, vc, d, H, rope_freq, pos_scale, rope, row, r.pos, r.page, ACB_LM_KV_PAGE,
                r.pos % ACB_LM_KV_PAGE, r.live);
}

// Paged admission pass (acb_lm_admit_prompt in a paged session): what the EPI_QKV_PF / EPI_QKV_PF_ROPE epilogue does, through
// the page table.
__global__ void __launch_bounds__(256) lm_qkv_pf_paged_kernel(const float* __restrict__ qkv, const int* __restrict__ P,
                                                              float* __restrict__ q32, __half* __restrict__ kc,
                                                              __half* __restrict__ vc, int d, int H, int rows_real,
                                                              const float* __restrict__ rope_freq, float pos_scale, bool rope,
                                                              const int* __restrict__ table, int pages_per_row, int r0,
                                                              int row_stride) {
    const int row = blockIdx.x;
    const PassRow r = pass_row(P, row, rows_real, r0, row_stride);
    const int page = table[r.trow * pages_per_row + r.pos / ACB_LM_KV_PAGE];
    qkv_f16_row(qkv + (size_t)row * 3 * d, q32, kc, vc, d, H, rope_freq, pos_scale, rope, row, r.pos, page, ACB_LM_KV_PAGE,
                r.pos % ACB_LM_KV_PAGE, true);
}

// ------------------------------------------------------------------------------------------------ FP8 KV pool
// An FP8 paged session (acb_lm_begin_slots_paged_fp8) keeps each 64-value K or V vector (one position of one head of one
// layer in one row) as 64 e4m3 codes in the pool [L][n_pages][H][ACB_LM_KV_PAGE][64] (uint8) and one fp32 scale in
// [L][n_pages][H][ACB_LM_KV_PAGE]; the vector reads back as code * scale.
struct Fp8Pool { uint8_t* k; uint8_t* v; float* ks; float* vs; };

// Quantize one vector, held by a warp as lane's values x0, x1 at dims 2 lane, 2 lane + 1: amax = max |x|,
// code = cvt.rn.satfinite.e4m3(x * (448 / amax)), scale = amax / 448 (both divisions correctly rounded, independent of
// compiler flags); amax == 0 gives zero codes and a zero scale.  codes points at the vector's 64 bytes.
__device__ __forceinline__ void quant_e4m3_warp(float x0, float x1, uint8_t* __restrict__ codes, float* __restrict__ scale,
                                                int lane) {
    const float amax = warp_max(fmaxf(fabsf(x0), fabsf(x1)));
    __nv_fp8x2_storage_t c = 0;
    float sc = 0.f;
    if (amax > 0.f) {
        const float inv = __fdiv_rn(448.f, amax);
        c = __nv_cvt_float2_to_fp8x2(make_float2(x0 * inv, x1 * inv), __NV_SATFINITE, __NV_E4M3);
        sc = __fdiv_rn(amax, 448.f);
    }
    reinterpret_cast<__nv_fp8x2_storage_t*>(codes)[lane] = c;
    if (lane == 0) *scale = sc;
}

// qkv_f16_row into an FP8 pool, for one row at cache position pos: q (rotated under rotary positions) to q32 in fp32, and,
// when `live`, each head's k (rotated) and v quantized into offset pos % page of `page`.  The values quantized are the fp32
// values the fp16 kernels round with __float2half_rn.  Warp w quantizes vectors w, w + 8, ... of the row's 2 H (K heads,
// then V heads).
__device__ __forceinline__ void qkv_fp8_row(const float* __restrict__ src, float* __restrict__ q32, Fp8Pool pool, int d, int H,
                                            const float* __restrict__ rope_freq, float pos_scale, bool rope, int row, int pos,
                                            int page, bool live) {
    for (int n = threadIdx.x; n < d; n += 256) {
        float v = src[n];
        if (rope) v = rope_rotate(rope_freq, pos_scale, half_round(v), half_round(src[n ^ 1]), n & 63, pos);
        q32[(size_t)row * d + n] = v;
    }
    if (!live) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int vec = warp; vec < 2 * H; vec += 8) {   // warp-uniform
        const int which = vec >= H, h = vec - which * H, i = 2 * lane;
        const float* s = src + (size_t)(1 + which) * d + h * 64;
        float x0 = s[i], x1 = s[i + 1];
        if (rope && !which) {
            const float a = half_round(x0), b = half_round(x1);
            x0 = rope_rotate(rope_freq, pos_scale, a, b, i, pos);
            x1 = rope_rotate(rope_freq, pos_scale, b, a, i + 1, pos);
        }
        const size_t at = ((size_t)page * H + h) * ACB_LM_KV_PAGE + pos % ACB_LM_KV_PAGE;
        quant_e4m3_warp(x0, x1, (which ? pool.v : pool.k) + at * 64, (which ? pool.vs : pool.ks) + at, lane);
    }
}

// lm_qkv_slot_paged_kernel into an FP8 pool (one layer's codes and scales in `pool`).
__global__ void __launch_bounds__(256) lm_qkv_slot_paged_fp8_kernel(const float* __restrict__ qkv, const int* __restrict__ slot_state,
                                                                    float* __restrict__ q32, Fp8Pool pool, int d, int H, int slots,
                                                                    const float* __restrict__ rope_freq, float pos_scale, bool rope,
                                                                    const int* __restrict__ table, int pages_per_row) {
    const int row = blockIdx.x;
    const SlotRow r = slot_row(slot_state, slots, row, table, pages_per_row);
    qkv_fp8_row(qkv + (size_t)row * 3 * d, q32, pool, d, H, rope_freq, pos_scale, rope, row, r.pos, r.page, r.live);
}

// lm_qkv_pf_paged_kernel into an FP8 pool.
__global__ void __launch_bounds__(256) lm_qkv_pf_paged_fp8_kernel(const float* __restrict__ qkv, const int* __restrict__ P,
                                                                  float* __restrict__ q32, Fp8Pool pool, int d, int H, int rows_real,
                                                                  const float* __restrict__ rope_freq, float pos_scale, bool rope,
                                                                  const int* __restrict__ table, int pages_per_row, int r0,
                                                                  int row_stride) {
    const int row = blockIdx.x;
    const PassRow r = pass_row(P, row, rows_real, r0, row_stride);
    const int page = table[r.trow * pages_per_row + r.pos / ACB_LM_KV_PAGE];
    qkv_fp8_row(qkv + (size_t)row * 3 * d, q32, pool, d, H, rope_freq, pos_scale, rope, row, r.pos, page, true);
}

// ------------------------------------------------------------------------------------------------ attention (1 query)
struct AttnParams {
    const float* q; int q_nsplit; size_t q_split_stride;  // q[s][row][d] fp32 partial sums
    const __half* kc; const __half* vc; __half* out;
    int H, d, cache_len; const int* pos; int fixed_len; float scale;
    int rows_real;                // prefill (PF kernels): rows of the generation
    int row_stride;               // prefill (PF kernels): row r of the generation is cache row r * row_stride of kc / vc
};

constexpr int ATT_WARPS = 8;

struct OnlineSM { float m, l, acc[8]; };
__device__ __forceinline__ void osm_merge(OnlineSM& a, float m2, float l2, const float (&acc2)[8]) {
    const float mn = fmaxf(a.m, m2);
    const float ca = a.m == -INFINITY ? 0.f : __expf(a.m - mn), cb = m2 == -INFINITY ? 0.f : __expf(m2 - mn);
    a.l = a.l * ca + l2 * cb;
#pragma unroll
    for (int e = 0; e < 8; ++e) a.acc[e] = a.acc[e] * ca + acc2[e] * cb;
    a.m = mn;
}

// Where position pp of a row's K/V lies, in 64-value vectors from the head's position 0: a contiguous cache row holds its
// positions in order; a paged row holds position pp at offset pp % ACB_LM_KV_PAGE of page pt[pp / ACB_LM_KV_PAGE], a page
// being [H][ACB_LM_KV_PAGE] vectors.  A page holds whole groups of the positions one warp instruction covers (4 in fp16,
// 8 in FP8), so no lane's 16-byte copy crosses a page.
struct RowAt {
    __device__ __forceinline__ size_t operator()(int pp) const { return (size_t)pp; }
};
struct PagedAt {
    const int* pt; int H;
    __device__ __forceinline__ size_t operator()(int pp) const {
        return (size_t)pt[pp / ACB_LM_KV_PAGE] * H * ACB_LM_KV_PAGE + pp % ACB_LM_KV_PAGE;
    }
};

// A paged attention CTA stages the first ceil(n / ACB_LM_KV_PAGE) entries (at most ACB_LM_MAX_PAGES_PER_ROW) of its page-table
// row trow in shared memory, behind one barrier.
__device__ __forceinline__ PagedAt stage_pages(const int* __restrict__ table, int pages_per_row, int trow, int n, int H) {
    __shared__ int pt[ACB_LM_MAX_PAGES_PER_ROW];
    for (int i = threadIdx.x; i < (n + ACB_LM_KV_PAGE - 1) / ACB_LM_KV_PAGE; i += ATT_WARPS * 32) pt[i] = table[trow * pages_per_row + i];
    __syncthreads();
    return {pt, H};
}

// The rows of a slot that is not ACTIVE attend to no key: the CTA (query row qrow, head blockIdx.x) writes zeros.
__device__ __forceinline__ void attn2_zero(const AttnParams& p, int qrow) {
    if (threadIdx.x < 64) p.out[(size_t)qrow * p.d + blockIdx.x * 64 + threadIdx.x] = __float2half_rn(0.f);
}

// The end of every self-attention CTA: each warp's merged online-softmax state (running max m, sum l, and E output dims per
// lane at sl * E, held by the lanes with `writer` set) goes to shared memory, and thread t < 64 merges the 8 warps for output
// dim t of the head, stored at out[t].
template <int E>
__device__ __forceinline__ void attn2_merge_store(float m, float l, const float (&acc)[E], bool writer, int sl,
                                                  __half* __restrict__ out) {
    __shared__ float wm[ATT_WARPS], wl[ATT_WARPS], wacc[ATT_WARPS][64];
    const int tid = threadIdx.x, warp = tid >> 5;
    if (writer) {
        if (sl == 0) { wm[warp] = m; wl[warp] = l; }
#pragma unroll
        for (int e = 0; e < E; ++e) wacc[warp][sl * E + e] = acc[e];
    }
    __syncthreads();
    if (tid < 64) {
        float mx = wm[0];
#pragma unroll
        for (int w = 1; w < ATT_WARPS; ++w) mx = fmaxf(mx, wm[w]);
        float lt = 0.f, o = 0.f;
#pragma unroll
        for (int w = 0; w < ATT_WARPS; ++w) {
            const float cw = wm[w] == -INFINITY ? 0.f : __expf(wm[w] - mx);
            lt = fmaf(wl[w], cw, lt);
            o = fmaf(wacc[w][tid], cw, o);
        }
        out[tid] = __float2half_rn(o / lt);
    }
}

// Self attention for one query token over an fp16 cache: CTA = (query row, head), 8 warps, ONE pass over K and V with an
// online softmax.  A warp instruction covers 4 consecutive cache positions (4 x 128 B = 512 contiguous bytes), 8 lanes share
// a position (8 dims each).  Every lane copies its 16-byte slices of K and V with cp.async into a private slot of a per-warp
// shared-memory ring, ATT2_DEPTH iterations deep, and reads them back (its own 32 bytes) one iteration at a time: up to
// 8 x 32 bytes per lane stay outstanding continuously, in shared memory instead of registers.
// Every instance runs this one body: query row qrow (of p.q and p.out) attends to positions [0, n) of the K/V whose head
// starts `head` vectors into p.kc / p.vc, position pp at(pp) vectors further (RowAt or PagedAt).  So the sums, and their
// order, are the same whatever the layout, and a paged session's results are bit-identical to a contiguous one's.
constexpr int ATT2_DEPTH = 8;
constexpr int ATT2_SMEM = ATT_WARPS * ATT2_DEPTH * 1024;   // the ring, 64 KB
template <class At>
__device__ __forceinline__ void attn2_body(const AttnParams& p, int qrow, int n, size_t head, At at) {
    extern __shared__ __align__(16) unsigned char att2sm[];   // [warp][depth][K | V][32 lanes][16 B]
    const int h = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int sl = lane & 7, pg = lane >> 3;
    const __half* kb = p.kc + (head * 64 + sl * 8);
    const __half* vb = p.vc + (head * 64 + sl * 8);
    const uint32_t ring = smem_u32(att2sm) + (uint32_t)(warp * ATT2_DEPTH * 1024 + lane * 16);
    // iteration k of this warp covers positions (k * 8 + warp) * 4 + pg
    const int n_it = (n + 31 - warp * 4) / 32 > 0 ? (n - warp * 4 + 31) / 32 : 0;   // iterations with at least one live position group
    auto issue = [&](int k) {
        if (k < n_it) {
            const int pp = (k * ATT_WARPS + warp) * 4 + pg;
            if (pp < n) {
                const uint32_t d = ring + (uint32_t)((k % ATT2_DEPTH) * 1024);
                const size_t o = at(pp) * 64;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(kb + o) : "memory");
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 512u), "l"(vb + o) : "memory");
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
#pragma unroll
    for (int k = 0; k < ATT2_DEPTH - 1; ++k) issue(k);

    float q[8];
    {
        const float4* qp = reinterpret_cast<const float4*>(p.q + (size_t)qrow * p.d + h * 64 + sl * 8);
        const float4 qa = qp[0], qb = qp[1];
        q[0] = half_round(qa.x) * p.scale; q[1] = half_round(qa.y) * p.scale; q[2] = half_round(qa.z) * p.scale;
        q[3] = half_round(qa.w) * p.scale; q[4] = half_round(qb.x) * p.scale; q[5] = half_round(qb.y) * p.scale;
        q[6] = half_round(qb.z) * p.scale; q[7] = half_round(qb.w) * p.scale;
    }
    OnlineSM st;
    st.m = -INFINITY; st.l = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) st.acc[e] = 0.f;

    for (int k = 0; k < n_it; ++k) {                 // warp-uniform trip count (the shuffles need all 32 lanes)
        issue(k + ATT2_DEPTH - 1);
        asm volatile("cp.async.wait_group %0;" ::"n"(ATT2_DEPTH - 1) : "memory");   // iteration k's copies of this lane have landed
        const int pp = (k * ATT_WARPS + warp) * 4 + pg;
        const uint32_t sa = ring + (uint32_t)((k % ATT2_DEPTH) * 1024);
        uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
        if (pp < n) {
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(kv.x), "=r"(kv.y), "=r"(kv.z), "=r"(kv.w) : "r"(sa));
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(vv.x), "=r"(vv.y), "=r"(vv.z), "=r"(vv.w) : "r"(sa + 512u));
        }
        const __half2* k2 = reinterpret_cast<const __half2*>(&kv);
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(k2[e]);
            s = fmaf(q[2 * e], f.x, s);
            s = fmaf(q[2 * e + 1], f.y, s);
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        if (pp < n) {
            const float mn = fmaxf(st.m, s);
            const float corr = __expf(st.m - mn);   // exp(-inf) = 0 on the first position
            const float pw = __expf(s - mn);
            st.l = st.l * corr + pw;
            const __half2* v2 = reinterpret_cast<const __half2*>(&vv);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __half22float2(v2[e]);
                st.acc[2 * e] = fmaf(pw, f.x, st.acc[2 * e] * corr);
                st.acc[2 * e + 1] = fmaf(pw, f.y, st.acc[2 * e + 1] * corr);
            }
            st.m = mn;
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    // merge the 4 position groups of the warp, then the warps
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, st.m, o), l2 = __shfl_xor_sync(0xffffffffu, st.l, o);
        float a2[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) a2[e] = __shfl_xor_sync(0xffffffffu, st.acc[e], o);
        osm_merge(st, m2, l2, a2);
    }
    attn2_merge_store(st.m, st.l, st.acc, pg == 0, sl, p.out + (size_t)qrow * p.d + h * 64);
}

// The decode step of generate (n = p.fixed_len, or p.pos[0] + 1) and prompt prefill.
// PF (prompt prefill): blockIdx.y is a (token, row) pair tok * rows_real + r; the query at position pos + tok attends to the
// cache of row r up to and including its own position (the QKV GEMM of the same pass has already appended every token of the
// pass: causal within the chunk); row r is cache row r * row_stride.
template <bool PF>
__global__ void __launch_bounds__(ATT_WARPS * 32) lm_attn2_kernel(AttnParams p) {
    const int qrow = blockIdx.y, row = PF ? qrow % p.rows_real * p.row_stride : qrow, tok = PF ? qrow / p.rows_real : 0;
    const int n = p.fixed_len > 0 ? p.fixed_len : p.pos[0] + tok + 1;
    attn2_body(p, qrow, n, ((size_t)row * p.H + blockIdx.x) * p.cache_len, RowAt{});
}

// Slot mode: each row at its own slot's position.  Row r of slot r % slots (p.rows_real = slots) attends to its slot's cache
// positions [0, prefix + pos]: the condition prefix and the columns so far.
__global__ void __launch_bounds__(ATT_WARPS * 32) lm_attn2_slot_kernel(AttnParams p, const int* __restrict__ slot_state) {
    const int qrow = blockIdx.y;
    const SlotRow r = slot_row(slot_state, p.rows_real, qrow, nullptr, 0);
    if (!r.live) { attn2_zero(p, qrow); return; }   // block-uniform
    attn2_body(p, qrow, r.pos + 1, ((size_t)qrow * p.H + blockIdx.x) * p.cache_len, RowAt{});
}

// Paged session (acb_lm_begin_slots_paged): lm_attn2_slot_kernel with p.kc / p.vc the layer's page pool.
__global__ void __launch_bounds__(ATT_WARPS * 32) lm_attn2_slot_paged_kernel(AttnParams p, const int* __restrict__ slot_state,
                                                                          const int* __restrict__ table, int pages_per_row) {
    const int qrow = blockIdx.y;
    const SlotRow r = slot_row(slot_state, p.rows_real, qrow, nullptr, 0);
    if (!r.live) { attn2_zero(p, qrow); return; }   // block-uniform
    attn2_body(p, qrow, r.pos + 1, (size_t)blockIdx.x * ACB_LM_KV_PAGE, stage_pages(table, pages_per_row, qrow, r.pos + 1, p.H));
}

// Paged admission pass (acb_lm_admit_prompt in a paged session): lm_attn2_kernel<true> reading K and V through the page table.
// The query of pass row qrow attends to positions [0, its own] of its page-table row (the pass's own positions are already
// appended: lm_qkv_pf_paged_kernel ran before).
__global__ void __launch_bounds__(ATT_WARPS * 32) lm_attn2_pf_paged_kernel(AttnParams p, const int* __restrict__ table,
                                                                        int pages_per_row, int r0) {
    const int qrow = blockIdx.y;
    const PassRow r = pass_row(p.pos, qrow, p.rows_real, r0, p.row_stride);
    attn2_body(p, qrow, r.pos + 1, (size_t)blockIdx.x * ACB_LM_KV_PAGE, stage_pages(table, pages_per_row, r.trow, r.pos + 1, p.H));
}

// Self attention over an FP8 pool: attn2_body's CTA (query row, head), online softmax and cp.async ring, with a lane's
// 16-byte copy holding 16 e4m3 codes: 4 lanes share a position (16 dims each), a warp instruction covers 8 consecutive
// positions, and iteration k of a warp covers positions (k * 8 + warp) * 8 + pg.  Lanes 0 and 1 of a position also copy its
// K and V scale into the stage.  Each lane dots its 16 codes (exact in fp16) with q in an fp32 FMA chain, the 4 lanes add in
// a 2-level shuffle tree, and the sum is multiplied by the K scale; the V scale multiplies the softmax weight before it
// scales the codes.  Query row qrow attends to positions [0, n) of the page-table row staged in `at`.
constexpr int ATT2F8_STAGE = 1024 + 64;   // per warp and stage: K codes, V codes [32 lanes][16 B], scales [8 positions][K, V]
constexpr int ATT2F8_SMEM = ATT_WARPS * ATT2_DEPTH * ATT2F8_STAGE;
__device__ __forceinline__ void attn2_paged_fp8_body(const AttnParams& p, const Fp8Pool& pool, int qrow, int n, PagedAt at) {
    extern __shared__ __align__(16) unsigned char att2sm[];   // [warp][depth][K | V | scales]
    const int h = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int sl = lane & 3, pg = lane >> 2;
    // position pp: codes at at(pp) * 64 + base, scales at at(pp) + h * page
    const uint8_t* kb = pool.k + (size_t)h * ACB_LM_KV_PAGE * 64 + sl * 16;
    const uint8_t* vb = pool.v + (size_t)h * ACB_LM_KV_PAGE * 64 + sl * 16;
    const float* sb = (sl ? pool.vs : pool.ks) + (size_t)h * ACB_LM_KV_PAGE;
    const uint32_t ring = smem_u32(att2sm) + (uint32_t)(warp * ATT2_DEPTH * ATT2F8_STAGE);
    const int n_it = n > warp * 8 ? (n - warp * 8 + 63) / 64 : 0;   // iterations with at least one live position group
    auto issue = [&](int k) {
        if (k < n_it) {
            const int pp = (k * ATT_WARPS + warp) * 8 + pg;
            if (pp < n) {
                const uint32_t st = ring + (uint32_t)((k % ATT2_DEPTH) * ATT2F8_STAGE);
                const size_t o = at(pp);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(st + lane * 16), "l"(kb + o * 64) : "memory");
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(st + 512u + lane * 16), "l"(vb + o * 64) : "memory");
                if (sl < 2)
                    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(st + 1024u + pg * 8 + sl * 4), "l"(sb + o)
                                 : "memory");
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
#pragma unroll
    for (int k = 0; k < ATT2_DEPTH - 1; ++k) issue(k);

    float q[16];
    {
        const float4* qp = reinterpret_cast<const float4*>(p.q + (size_t)qrow * p.d + h * 64 + sl * 16);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const float4 a = qp[c];
            q[4 * c] = half_round(a.x) * p.scale; q[4 * c + 1] = half_round(a.y) * p.scale;
            q[4 * c + 2] = half_round(a.z) * p.scale; q[4 * c + 3] = half_round(a.w) * p.scale;
        }
    }
    float m = -INFINITY, l = 0.f, acc[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) acc[e] = 0.f;

    for (int k = 0; k < n_it; ++k) {                 // warp-uniform trip count (the shuffles need all 32 lanes)
        __syncwarp();                                // every lane has read stage k - 1 before issue() refills it
        issue(k + ATT2_DEPTH - 1);
        asm volatile("cp.async.wait_group %0;" ::"n"(ATT2_DEPTH - 1) : "memory");   // iteration k's copies of this lane have landed
        __syncwarp();                                // and the scales lanes 0 / 1 of each position copied are visible
        const int pp = (k * ATT_WARPS + warp) * 8 + pg;
        const uint32_t sa = ring + (uint32_t)((k % ATT2_DEPTH) * ATT2F8_STAGE);
        uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
        float ksc = 0.f, vsc = 0.f;
        if (pp < n) {
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(kv.x), "=r"(kv.y), "=r"(kv.z), "=r"(kv.w) : "r"(sa + lane * 16));
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(vv.x), "=r"(vv.y), "=r"(vv.z), "=r"(vv.w)
                         : "r"(sa + 512u + lane * 16));
            asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(ksc), "=f"(vsc) : "r"(sa + 1024u + pg * 8));
        }
        const __nv_fp8x2_storage_t* k2 = reinterpret_cast<const __nv_fp8x2_storage_t*>(&kv);
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float2 f = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(k2[e], __NV_E4M3)));
            s = fmaf(q[2 * e], f.x, s);
            s = fmaf(q[2 * e + 1], f.y, s);
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        s *= ksc;
        if (pp < n) {
            const float mn = fmaxf(m, s);
            const float corr = __expf(m - mn);      // exp(-inf) = 0 on the first position
            const float pw = __expf(s - mn);
            l = l * corr + pw;
            const float pv = pw * vsc;
            const __nv_fp8x2_storage_t* v2 = reinterpret_cast<const __nv_fp8x2_storage_t*>(&vv);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float2 f = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(v2[e], __NV_E4M3)));
                acc[2 * e] = fmaf(pv, f.x, acc[2 * e] * corr);
                acc[2 * e + 1] = fmaf(pv, f.y, acc[2 * e + 1] * corr);
            }
            m = mn;
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    // merge the 8 position groups of the warp (xor 4, 8, 16), then the warps
#pragma unroll
    for (int o = 4; o <= 16; o <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, o), l2 = __shfl_xor_sync(0xffffffffu, l, o);
        const float mn = fmaxf(m, m2);
        const float ca = m == -INFINITY ? 0.f : __expf(m - mn), cb = m2 == -INFINITY ? 0.f : __expf(m2 - mn);
        l = l * ca + l2 * cb;
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[e] = acc[e] * ca + __shfl_xor_sync(0xffffffffu, acc[e], o) * cb;
        m = mn;
    }
    attn2_merge_store(m, l, acc, pg == 0, sl, p.out + (size_t)qrow * p.d + h * 64);
}

// lm_attn2_slot_paged_kernel over an FP8 pool (one layer's codes and scales in `pool`).
__global__ void __launch_bounds__(ATT_WARPS * 32) lm_attn2_slot_paged_fp8_kernel(AttnParams p, Fp8Pool pool,
                                                                              const int* __restrict__ slot_state,
                                                                              const int* __restrict__ table, int pages_per_row) {
    const int qrow = blockIdx.y;
    const SlotRow r = slot_row(slot_state, p.rows_real, qrow, nullptr, 0);
    if (!r.live) { attn2_zero(p, qrow); return; }   // block-uniform
    attn2_paged_fp8_body(p, pool, qrow, r.pos + 1, stage_pages(table, pages_per_row, qrow, r.pos + 1, p.H));
}

// lm_attn2_pf_paged_kernel over an FP8 pool.
__global__ void __launch_bounds__(ATT_WARPS * 32) lm_attn2_pf_paged_fp8_kernel(AttnParams p, Fp8Pool pool,
                                                                            const int* __restrict__ table, int pages_per_row,
                                                                            int r0) {
    const int qrow = blockIdx.y;
    const PassRow r = pass_row(p.pos, qrow, p.rows_real, r0, p.row_stride);
    attn2_paged_fp8_body(p, pool, qrow, r.pos + 1, stage_pages(table, pages_per_row, r.trow, r.pos + 1, p.H));
}

// Cross attention over the (short) text condition: one WARP per (row, head), lane = text position for the scores,
// lane = 2 output dims for the weighted sum.  K/V were computed once per generate() (acb_lm_begin).
// The warp's query row `row`, head h attends to the first n >= 1 text positions of cache row `crow`.
__device__ __forceinline__ void cross_attn_body(const AttnParams& p, int row, int h, int crow, int n) {
    __shared__ float qs[8][64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    {
        const float* qp = p.q + (size_t)row * p.d + h * 64 + lane * 2;
        float2 part[ACB_LM_MAX_SPLIT];
#pragma unroll
        for (int s = 0; s < ACB_LM_MAX_SPLIT; ++s)   // independent loads, fixed summation order
            part[s] = s < p.q_nsplit ? *reinterpret_cast<const float2*>(qp + s * p.q_split_stride) : make_float2(0.f, 0.f);
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int s = 0; s < ACB_LM_MAX_SPLIT; ++s) { a0 += part[s].x; a1 += part[s].y; }
        qs[warp][lane * 2] = half_round(a0) * p.scale;
        qs[warp][lane * 2 + 1] = half_round(a1) * p.scale;
    }
    __syncwarp();
    const size_t base = ((size_t)crow * p.H + h) * p.cache_len * 64;
    float mx = -INFINITY, l = 0.f, o0 = 0.f, o1 = 0.f;
    for (int t0 = 0; t0 < n; t0 += 32) {             // chunks of 32 text positions (online softmax across chunks)
        const int t = t0 + lane;
        float s = -INFINITY;
        if (t < n) {
            const uint4* kr = reinterpret_cast<const uint4*>(p.kc + base + (size_t)t * 64);
            s = 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 kk = kr[c];
                const __half2* k2 = reinterpret_cast<const __half2*>(&kk);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(k2[e]);
                    s = fmaf(qs[warp][c * 8 + 2 * e], f.x, s);
                    s = fmaf(qs[warp][c * 8 + 2 * e + 1], f.y, s);
                }
            }
        }
        const float cm = fmaxf(mx, warp_max(s));
        const float corr = mx == -INFINITY ? 0.f : __expf(mx - cm);
        const float pw = t < n ? __expf(s - cm) : 0.f;
        l = l * corr + warp_sum(pw);
        o0 *= corr; o1 *= corr;
        const int cnt = min(32, n - t0);
        for (int j = 0; j < cnt; ++j) {
            const float wj = __shfl_sync(0xffffffffu, pw, j);
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(p.vc + base + (size_t)(t0 + j) * 64 + lane * 2));
            o0 = fmaf(wj, f.x, o0);
            o1 = fmaf(wj, f.y, o1);
        }
        mx = cm;
    }
    *reinterpret_cast<__half2*>(p.out + (size_t)row * p.d + h * 64 + lane * 2) = __floats2half2_rn(o0 / l, o1 / l);
}

template <bool PF>
__global__ void __launch_bounds__(256) lm_cross_attn_kernel(AttnParams p, int rows) {
    const int pair = blockIdx.x * 8 + (threadIdx.x >> 5);   // (row, head) index
    if (pair >= rows * p.H) return;                         // warp-uniform
    const int row = pair / p.H, h = pair % p.H;
    cross_attn_body(p, row, h, PF ? row % p.rows_real * p.row_stride : row, p.fixed_len);   // K / V of the generation row
}

// Slot mode: row r attends to exactly its slot's own text length (p.rows_real = slots), not to a length shared by the batch,
// so a request's result does not depend on the other requests' conditions.  A slot never admitted (length 0) writes zeros.
__global__ void __launch_bounds__(256) lm_cross_attn_slot_kernel(AttnParams p, int rows, const int* __restrict__ slot_state) {
    const int pair = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (pair >= rows * p.H) return;
    const int row = pair / p.H, h = pair % p.H, lane = threadIdx.x & 31;
    const int n = slot_state[(row % p.rows_real) * ACB_LM_SLOT_STRIDE + ACB_SLOT_TEXT_LEN];
    if (n <= 0) {
        *reinterpret_cast<__half2*>(p.out + (size_t)row * p.d + h * 64 + lane * 2) = __floats2half2_rn(0.f, 0.f);
        return;
    }
    cross_attn_body(p, row, h, row, n);
}

// ------------------------------------------------------------------------------------------------ sampling
// Philox4x32-10 (counter-based; one 4-word block per 4 candidates) -> 24-bit uniforms -> Exponential(1).
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
        uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += W0;
        key.y += W1;
    }
    return ctr;
}
__device__ __forceinline__ float exp1_noise(uint64_t seed, uint32_t step, uint32_t stream, uint32_t i) {
    uint4 r = philox4x32_10(make_uint4(i >> 2, stream, step, 0x5a17u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    uint32_t w = (i & 3) == 0 ? r.x : ((i & 3) == 1 ? r.y : ((i & 3) == 2 ? r.z : r.w));
    float u = ((float)(w >> 8) + 0.5f) * (1.0f / 16777216.0f);  // (0,1), never 0 or 1
    return -logf(u);
}

struct SampleParams {
    const float* logits;  // [rows][n_q*card]
    const float* noise;   // [batch][n_q][card] or NULL
    float* logits_out;    // [batch][n_q][card] CFG-mixed logits or NULL
    int64_t* seq; const uint8_t* seq_mask; int* pos; int max_seq;  // in-loop write-back (seq may be NULL)
    int64_t* tokens;      // [batch][n_q] stand-alone output (may be NULL)
    int batch, rows, n_q, card, NP;
    int use_sampling, top_k; float temp, top_p, cfg_coef; uint64_t seed; uint32_t step;
    float cfg_coef_beta;   // rows == 3 * batch: double CFG (lm.py:362-376)
    int seq_off;           // condition-prefix length: cache position pos is sequence column pos - seq_off
};

// descending order, ties by ascending index
__device__ __forceinline__ bool before(float va, int ia, float vb, int ib) { return va > vb || (va == vb && ia < ib); }

// lm_sample_kernel and (SLOT) lm_sample_slot_kernel: CFG mix, sampling, first-max argmax and the write-back of block (k, b).
template <bool SLOT>
__device__ __forceinline__ void sample_impl(const SampleParams& p, int* slot_state) {
    extern __shared__ float sm[];
    float* pr = sm;                 // [card] logits -> probabilities
    float* sv = pr + p.card;        // [NP] sort values
    int* si = (int*)(sv + p.NP);    // [NP] sort indices
    __shared__ float red[3][32];
    __shared__ float bestv[32];
    __shared__ int besti[32];
    __shared__ float s_scalar;
    const int k = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, nt = blockDim.x;
    int* st = SLOT ? slot_state + b * ACB_LM_SLOT_STRIDE : nullptr;
    if (SLOT && st[ACB_SLOT_STATUS] != SLOT_ACTIVE) return;   // block-uniform
    const int card = p.card;
    const bool cfg = p.rows == 2 * p.batch, cfg3 = p.rows == 3 * p.batch;   // [cond; null] or [cond; style-only; null]
    const float* lc = p.logits + ((size_t)b * p.n_q + k) * card;
    const float* lu = p.logits + ((size_t)((cfg3 ? 2 : 1) * p.batch + b) * p.n_q + k) * card;
    const float* lw = p.logits + ((size_t)(p.batch + b) * p.n_q + k) * card;
    const int cur_pos = SLOT ? st[ACB_SLOT_POS] : (p.pos ? p.pos[0] : 0);   // read once: the last block to finish advances it
    const int col = cur_pos - p.seq_off;        // sequence column of the token this step consumed
    const uint32_t step = (SLOT || p.pos) ? (uint32_t)col : p.step;
    uint64_t slot_seed = 0;
    if constexpr (SLOT)
        slot_seed = (uint64_t)(uint32_t)st[ACB_SLOT_SEED_LO] | ((uint64_t)(uint32_t)st[ACB_SLOT_SEED_HI] << 32);

    for (int i = tid; i < card; i += nt) {
        float l = lc[i];
        if (cfg) { float u = lu[i]; l = u + (l - u) * p.cfg_coef; }   // lm.py:399
        else if (cfg3) { const float u = lu[i], w = lw[i]; l = u + p.cfg_coef * (w + p.cfg_coef_beta * (l - w) - u); }   // lm.py:372-376
        pr[i] = l;
        if (p.logits_out) p.logits_out[((size_t)b * p.n_q + k) * card + i] = l;
    }
    __syncthreads();

    const bool sampling = p.use_sampling && p.temp > 0.f;
    bool sorted_space = false;
    if (sampling) {
        float lm = -INFINITY;
        for (int i = tid; i < card; i += nt) { float l = pr[i] / p.temp; pr[i] = l; lm = fmaxf(lm, l); }
        const float m = block_max(lm, red[0]);
        float ls = 0.f;
        for (int i = tid; i < card; i += nt) { float e = expf(pr[i] - m); pr[i] = e; ls += e; }
        const float s = block_sum(ls, red[1]);
        for (int i = tid; i < card; i += nt) pr[i] = pr[i] / s;
        __syncthreads();
        const int kk = p.top_k > card ? card : p.top_k;
        if (p.top_p <= 0.f && kk > 0) {
            // utils.sample_top_k (utils/utils.py:108-122) keeps p >= the k-th largest probability and renormalises: only
            // that VALUE is needed, so instead of sorting (66 block barriers for 2048 candidates) select it exactly with
            // a 4-pass radix select on the bit patterns (non-negative floats order like their uint32 bits).
            __shared__ int hist[256];
            __shared__ int s_bin, s_rem;
            uint32_t prefix = 0u, mask = 0u;
            int remaining = kk;                     // rank (from the top) among the candidates matching prefix/mask
#pragma unroll 1
            for (int shift = 24; shift >= 0; shift -= 8) {
                for (int i = tid; i < 256; i += nt) hist[i] = 0;
                __syncthreads();
                for (int i = tid; i < card; i += nt) {
                    const uint32_t key = __float_as_uint(pr[i]);
                    if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1);
                }
                __syncthreads();
                if (tid == 0) {
                    int acc = 0, bin = 255;
                    for (; bin > 0; --bin) {
                        if (acc + hist[bin] >= remaining) break;
                        acc += hist[bin];
                    }
                    s_bin = bin; s_rem = remaining - acc;
                }
                __syncthreads();
                prefix |= (uint32_t)s_bin << shift;
                mask |= 255u << shift;
                remaining = s_rem;
            }
            const float kth = __uint_as_float(prefix);
            float ls2 = 0.f;
            for (int i = tid; i < card; i += nt) { float v = pr[i] >= kth ? pr[i] : 0.f; pr[i] = v; ls2 += v; }
            const float s2 = block_sum(ls2, red[2]);
            for (int i = tid; i < card; i += nt) pr[i] = pr[i] / s2;
            __syncthreads();
        } else if (p.top_p > 0.f || kk > 0) {
            for (int i = tid; i < p.NP; i += nt) { sv[i] = i < card ? pr[i] : -INFINITY; si[i] = i; }
            __syncthreads();
            for (int size = 2; size <= p.NP; size <<= 1)
                for (int j = size >> 1; j > 0; j >>= 1) {
                    for (int i = tid; i < p.NP; i += nt) {
                        const int l = i ^ j;
                        if (l > i) {
                            const bool fwd = (i & size) == 0;
                            float va = sv[i], vb = sv[l];
                            int ia = si[i], ib = si[l];
                            const bool ok = before(va, ia, vb, ib);
                            if (fwd ? !ok : ok) { sv[i] = vb; sv[l] = va; si[i] = ib; si[l] = ia; }
                        }
                    }
                    __syncthreads();
                }
            if (p.top_p > 0.f) {
                // utils.sample_top_p (utils/utils.py:125-141): sequential cumsum like torch's CPU kernel
                if (tid == 0) {
                    float cum = 0.f;
                    for (int i = 0; i < card; ++i) {
                        const float v = sv[i];
                        cum += v;
                        if (cum - v > p.top_p) sv[i] = 0.f;
                    }
                }
                __syncthreads();
                float ls2 = 0.f;
                for (int i = tid; i < card; i += nt) ls2 += sv[i];
                const float s2 = block_sum(ls2, red[2]);
                for (int i = tid; i < card; i += nt) pr[i] = sv[i] / s2;  // pr now lives in sorted space
                sorted_space = true;
                __syncthreads();
            } else {
                // utils.sample_top_k (utils/utils.py:108-122): keep p >= k-th largest, renormalise
                if (tid == 0) s_scalar = sv[kk - 1];
                __syncthreads();
                const float kth = s_scalar;
                float ls2 = 0.f;
                for (int i = tid; i < card; i += nt) { float v = pr[i] >= kth ? pr[i] : 0.f; pr[i] = v; ls2 += v; }
                const float s2 = block_sum(ls2, red[2]);
                for (int i = tid; i < card; i += nt) pr[i] = pr[i] / s2;
                __syncthreads();
            }
        }
        // torch.multinomial(num_samples=1): argmax_i p_i / q_i, q ~ Exponential(1)
        for (int i = tid; i < card; i += nt) {
            const float qn = p.noise ? p.noise[((size_t)b * p.n_q + k) * card + i]
                                     : exp1_noise(SLOT ? slot_seed : p.seed, step,
                                                  SLOT ? (uint32_t)k : (uint32_t)(b * p.n_q + k), (uint32_t)i);
            pr[i] = pr[i] / qn;
        }
        __syncthreads();
    }
    // first-max argmax over pr
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < card; i += nt) {
        const float v = pr[i];
        if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if ((tid & 31) == 0) { bestv[tid >> 5] = bv; besti[tid >> 5] = bi; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < (nt >> 5); ++w)
            if (bestv[w] > bv || (bestv[w] == bv && besti[w] < bi)) { bv = bestv[w]; bi = besti[w]; }
        if (bi == 0x7fffffff) bi = 0;
        int tok = sorted_space ? si[bi] : bi;
        if constexpr (SLOT) {
            const int off = col + 1;   // < the slot's seq_len while it is active
            const size_t at = ((size_t)b * p.n_q + k) * p.max_seq + off;
            if (!p.seq_mask[at]) tok = card;
            if (p.seq[at] == -1) p.seq[at] = tok;
            __threadfence();
            const int done = atomicAdd(st + ACB_SLOT_DONE, 1);
            if (done == p.n_q - 1) {   // the slot's last block: advance it, and finish it after its last column
                st[ACB_SLOT_DONE] = 0;
                st[ACB_SLOT_POS] = off;
                if (off >= st[ACB_SLOT_SEQ_LEN] - 1) st[ACB_SLOT_STATUS] = SLOT_FINISHED;
            }
        } else {
            if (p.tokens) p.tokens[(size_t)b * p.n_q + k] = tok;
            if (p.seq) {
                const int off = col + 1;
                if (off < p.max_seq) {
                    if (!p.seq_mask[(size_t)k * p.max_seq + off]) tok = card;            // lm.py:555-556
                    int64_t* dst = p.seq + ((size_t)b * p.n_q + k) * p.max_seq + off;
                    if (*dst == -1) *dst = tok;                                           // lm.py:559-562
                }
                // the last (b, k) block to get here advances the position: pos[1] counts finished blocks
                __threadfence();
                const int done = atomicAdd(p.pos + 1, 1);
                if (done == (int)(gridDim.x * gridDim.y) - 1) { p.pos[1] = 0; p.pos[0] = cur_pos + 1; }
            }
        }
    }
}

__global__ void __launch_bounds__(1024) lm_sample_kernel(SampleParams p) { sample_impl<false>(p, nullptr); }

// Slot mode's sampler: block (k, slot), slots not ACTIVE skipped.  Column, step and seed are the slot's own, and the noise is
// Philox stream k of (seed, column) -- what lm_sample_kernel draws for item 0 of a generation, so a request samples as if
// generated alone.  p.seq_mask is [slots][n_q][max_seq].  A known token (!= -1) stays, so a prompt written into the sequence
// is consumed one column per step.  The last of the slot's n_q blocks advances its position; writing column seq_len - 1
// finishes the slot.  The sampling options are the slot's own record in slot_sampling (written at admission), so the captured
// step serves requests with different options: every choice they drive (CFG coefficient, temperature, top-k radix select or
// top-p sort, argmax) is uniform over a block.
__global__ void __launch_bounds__(1024) lm_sample_slot_kernel(SampleParams p, int* __restrict__ slot_state,
                                                              const int* __restrict__ slot_sampling) {
    const int* rec = slot_sampling + blockIdx.y * ACB_LM_SLOT_SAMPLING_STRIDE;
    p.use_sampling = rec[0];
    p.temp = __int_as_float(rec[1]);
    p.top_k = rec[2];
    p.top_p = __int_as_float(rec[3]);
    p.cfg_coef = __int_as_float(rec[4]);
    sample_impl<true>(p, slot_state);
}

// Admission of a request's sampling options (the record lm_sample_slot_kernel reads).
__global__ void lm_slot_sampling_kernel(int* slot_sampling, int slot, int use_sampling, float temp, int top_k, float top_p,
                                        float cfg_coef) {
    int* rec = slot_sampling + slot * ACB_LM_SLOT_SAMPLING_STRIDE;
    rec[0] = use_sampling;
    rec[1] = __float_as_int(temp);
    rec[2] = top_k;
    rec[3] = __float_as_int(top_p);
    rec[4] = __float_as_int(cfg_coef);
}

// Cancellation: the slot is skipped from the next step on, as a slot never admitted.
__global__ void lm_slot_retire_kernel(int* slot_state, int slot) {
    slot_state[slot * ACB_LM_SLOT_STRIDE + ACB_SLOT_STATUS] = SLOT_INACTIVE;
}

// Admission: the slot starts at column 0 with its own sequence length, text length, condition-prefix length and seed.
__global__ void lm_slot_admit_kernel(int* slot_state, int slot, int seq_len, int text_len, int prefix_len, uint32_t seed_lo,
                                     uint32_t seed_hi) {
    int* st = slot_state + slot * ACB_LM_SLOT_STRIDE;
    st[ACB_SLOT_POS] = 0;
    st[ACB_SLOT_PREFIX] = prefix_len;
    st[ACB_SLOT_STATUS] = SLOT_ACTIVE;
    st[ACB_SLOT_SEQ_LEN] = seq_len;
    st[ACB_SLOT_TEXT_LEN] = text_len;
    st[ACB_SLOT_SEED_LO] = (int)seed_lo;
    st[ACB_SLOT_SEED_HI] = (int)seed_hi;
    st[ACB_SLOT_DONE] = 0;
}

// Paged session admission: the slot's two page-table rows (cond row r0, null row r1), n page ids each, passed by value.
struct PageList { int ids[2 * ACB_LM_MAX_PAGES_PER_ROW]; };
__global__ void lm_page_table_kernel(int* table, int pages_per_row, int r0, int r1, int n, PageList pl) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        table[r0 * pages_per_row + i] = pl.ids[i];
        table[r1 * pages_per_row + i] = pl.ids[n + i];
    }
}

// Paged session admission of a condition prefix: positions [0, P) of the staging cache [L][2][H][max_prefix][64] (its row 0 is
// the slot's cond row r0, row 1 its null row r1) copied into the rows' pages, 16 bytes per thread.
__global__ void lm_prefix_scatter_kernel(const __half* __restrict__ sk, const __half* __restrict__ sv, __half* __restrict__ pk,
                                         __half* __restrict__ pv, const int* __restrict__ table, int pages_per_row, int r0,
                                         int r1, int H, int max_prefix, int P, size_t pool_layer, size_t total) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % 8);
    size_t t = i / 8;
    const int pos = (int)(t % P); t /= P;
    const int h = (int)(t % H); t /= H;
    const int j = (int)(t % 2);
    const size_t l = t / 2;
    const size_t src = (((l * 2 + j) * H + h) * max_prefix + pos) * 64 + c * 8;
    const int page = table[(j ? r1 : r0) * pages_per_row + pos / ACB_LM_KV_PAGE];
    const size_t dst = l * pool_layer + (((size_t)page * H + h) * ACB_LM_KV_PAGE + pos % ACB_LM_KV_PAGE) * 64 + c * 8;
    *reinterpret_cast<uint4*>(pk + dst) = *reinterpret_cast<const uint4*>(sk + src);
    *reinterpret_cast<uint4*>(pv + dst) = *reinterpret_cast<const uint4*>(sv + src);
}

// lm_prefix_scatter_kernel into an FP8 pool (pool: layer 0's codes and scales; pool_layer: elements of one layer's scales):
// one warp per staged fp16 vector (K or V of one position of one head of one layer in one row), quantized as the step
// quantizes its own.
__global__ void lm_prefix_scatter_fp8_kernel(const __half* __restrict__ sk, const __half* __restrict__ sv, Fp8Pool pool,
                                             const int* __restrict__ table, int pages_per_row, int r0, int r1, int H,
                                             int max_prefix, int P, size_t pool_layer, size_t n_vec) {
    const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n_vec) return;   // warp-uniform
    size_t t = i;
    const int which = (int)(t % 2); t /= 2;
    const int pos = (int)(t % P); t /= P;
    const int h = (int)(t % H); t /= H;
    const int j = (int)(t % 2);
    const size_t l = t / 2;
    const size_t src = (((l * 2 + j) * H + h) * max_prefix + pos) * 64 + 2 * lane;
    const float2 x = __half22float2(*reinterpret_cast<const __half2*>((which ? sv : sk) + src));
    const int page = table[(j ? r1 : r0) * pages_per_row + pos / ACB_LM_KV_PAGE];
    const size_t at = l * pool_layer + ((size_t)page * H + h) * ACB_LM_KV_PAGE + pos % ACB_LM_KV_PAGE;
    quant_e4m3_warp(x.x, x.y, (which ? pool.v : pool.k) + at * 64, (which ? pool.vs : pool.ks) + at, lane);
}

__global__ void lm_f32_to_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, size_t n_valid, size_t n_total) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_total) dst[i] = __float2half_rn(i < n_valid ? src[i] : 0.f);
}

// ------------------------------------------------------------------------------------------------ host side
struct acb_lm {
    acb_lm_config cfg;
    acb_lm_weights w;
    acb_lm_buffers buf;
    acb_lm_sampling samp;
    cudaStream_t capture_stream = nullptr;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    int batch = 0, rows = 0, rows_pad = 0, text_len = 0, seq_len = 0, sms = 132;
    int slots = 0;                 // slot mode (acb_lm_begin_slots): batch = slots, rows = 2 * slots, per-slot device state
    int prefix_len = 0;            // condition-prefix positions in front of the tokens in the KV cache
    const float* prefix = nullptr; // [rows][prefix_len][d] fp32, set only while acb_lm_begin_prefix / _admit_prefix enqueue passes
    // set only while acb_lm_admit_prefix enqueues a slot's prefix passes (-1 otherwise): the passes run on that slot's two
    // rows (cache rows pf_slot and slots + pf_slot) with its own text length, as a generation of batch 1 with CFG would
    int pf_slot = -1, pf_text_len = 0;
    int launches = 0;
    bool has_cross = false;
    // paged handle (created with buffers.k_cache == NULL): the session's self-attention cache is the page pool of
    // acb_lm_begin_slots_paged, [L][n_pages][H][ACB_LM_KV_PAGE][64], and an admission's prefix passes run into the staging
    // cache [L][2][H][max_prefix][64] of the slot's two rows
    bool paged = false;
    __half* pool_k = nullptr; __half* pool_v = nullptr;
    int n_pages = 0, pages_per_row = 0, max_prefix = 0;
    int* page_table = nullptr;
    __half* stage_k = nullptr; __half* stage_v = nullptr;
    // FP8 paged session (acb_lm_begin_slots_paged_fp8): pool_k / pool_v hold e4m3 codes and pool_ks / pool_vs the scales
    // [L][n_pages][H][ACB_LM_KV_PAGE]
    bool fp8 = false;
    float* pool_ks = nullptr; float* pool_vs = nullptr;
    // wide GEMM (max_rows > 64): one map per stacked weight matrix [L * N][K] (encoded by acb_lm_create) and per activation
    // buffer [rows][K] of the current generation (encoded by acb_lm_begin_prefix)
    CUtensorMap wmap[7];
    CUtensorMap xmap_h16, xmap_a16, xmap_f16;
    bool w8 = false;   // weight_dtype 1: e4m3 per-layer matrices with row scales (lm_gemm_fp8_kernel, lm_gemm_wide_fp8_kernel)
};
enum { WM_QKV = 0, WM_O, WM_CQ, WM_CO, WM_FF1, WM_FF2, WM_HEADS };

static int nt_for_rows(int rows) { return rows <= 8 ? 1 : (rows <= 16 ? 2 : (rows <= 32 ? 4 : 8)); }

static size_t gemm_smem_bytes(int nt, int kslice, int ft2 = 1, bool w8 = false) {
    return (size_t)16 * ft2 * gemm_pitch(kslice, w8) + 16 + (size_t)4 * 16 * ft2 * (8 * nt + 1) * sizeof(float);
}
constexpr int GEMM_MAX_SMEM = 120 * 1024;

// wscale: the row scales of an FP8 matrix (p.W holds its codes), NULL for fp16
template <int EPI, int FT2>
static int launch_gemm_ft(int nt, const GemmParams& p, int nsplit, cudaStream_t s, const float* wscale) {
    dim3 grid(p.N / (16 * FT2), nsplit);
    const size_t smem = gemm_smem_bytes(nt, p.kslice, FT2, wscale != nullptr);
    ACB_REQUIRE(smem <= (size_t)GEMM_MAX_SMEM && p.N % (16 * FT2) == 0, "lm_gemm: tile does not fit (N=%d kslice=%d ft2=%d)", p.N, p.kslice, FT2);
    if (wscale) {
        switch (nt) {
            case 1: lm_gemm_fp8_kernel<1, EPI, FT2><<<grid, 128, smem, s>>>(p, wscale); break;
            case 2: lm_gemm_fp8_kernel<2, EPI, FT2><<<grid, 128, smem, s>>>(p, wscale); break;
            case 4: lm_gemm_fp8_kernel<4, EPI, FT2><<<grid, 128, smem, s>>>(p, wscale); break;
            default: lm_gemm_fp8_kernel<8, EPI, FT2><<<grid, 128, smem, s>>>(p, wscale); break;
        }
    } else {
        switch (nt) {
            case 1: lm_gemm_kernel<1, EPI, FT2><<<grid, 128, smem, s>>>(p); break;
            case 2: lm_gemm_kernel<2, EPI, FT2><<<grid, 128, smem, s>>>(p); break;
            case 4: lm_gemm_kernel<4, EPI, FT2><<<grid, 128, smem, s>>>(p); break;
            default: lm_gemm_kernel<8, EPI, FT2><<<grid, 128, smem, s>>>(p); break;
        }
    }
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}
template <int EPI>
static int launch_gemm(int nt, const GemmParams& p, int nsplit, cudaStream_t s, int ft2 = 1, const float* wscale = nullptr) {
    if (ft2 == 2) {
        if constexpr (EPI == EPI_CROSSKV || EPI == EPI_QKV_PF || EPI == EPI_QKV_PF_ROPE) { acb_set_error("lm_gemm: this epilogue uses 16-feature tiles"); return ACB_ERR_INVALID; }
        else return launch_gemm_ft<EPI, 2>(nt, p, nsplit, s, wscale);
    }
    return launch_gemm_ft<EPI, 1>(nt, p, nsplit, s, wscale);
}

template <int NT, int EPI, int FT2>
static cudaError_t gemm_attr_one(bool w8) {
    const void* f = w8 ? (const void*)lm_gemm_fp8_kernel<NT, EPI, FT2> : (const void*)lm_gemm_kernel<NT, EPI, FT2>;
    cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_MAX_SMEM);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(f, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
}
template <int EPI>
static cudaError_t gemm_attr_all(bool w8 = false) {
    cudaError_t e;
    if ((e = gemm_attr_one<1, EPI, 1>(w8)) != cudaSuccess) return e;
    if ((e = gemm_attr_one<2, EPI, 1>(w8)) != cudaSuccess) return e;
    if ((e = gemm_attr_one<4, EPI, 1>(w8)) != cudaSuccess) return e;
    if ((e = gemm_attr_one<8, EPI, 1>(w8)) != cudaSuccess) return e;
    if constexpr (EPI != EPI_CROSSKV && EPI != EPI_QKV_PF && EPI != EPI_QKV_PF_ROPE) {
        if ((e = gemm_attr_one<1, EPI, 2>(w8)) != cudaSuccess) return e;
        if ((e = gemm_attr_one<2, EPI, 2>(w8)) != cudaSuccess) return e;
        if ((e = gemm_attr_one<4, EPI, 2>(w8)) != cudaSuccess) return e;
        if ((e = gemm_attr_one<8, EPI, 2>(w8)) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// 32-feature tiles for a GEMM?  Only the big ones (their k-loop is bound by activation re-reads), only when the grid
// still covers ~90 % of the SMs and the 32-row weight slab fits.  ACB_LM_FT32=0 turns it off.
static int pick_ft2(int N, int K, int nsplit, int kslice, int nt, int sms) {
    const char* e = getenv("ACB_LM_FT32");
    const bool enabled = !(e && e[0] == '0');
    if (!enabled || N % 32 != 0 || (size_t)N * K < ((size_t)2 << 20)) return 1;   // d x d at d = 1536 qualifies (2.36 M weights)
    if ((N / 32) * nsplit * 10 < sms * 9) return 1;
    if (gemm_smem_bytes(nt, kslice, 2) > (size_t)GEMM_MAX_SMEM) return 1;
    return 2;
}

// K-slices per GEMM: the slab a CTA stages (16 x kslice fp16) must fit ~64 KB of shared memory, and when the
// consumer can reduce partial sums (allow_split) the matrix is cut further until there are >= 2 CTAs per SM.
// Returns nsplit (grid.y) and sets *kslice (a multiple of 32 elements).
static int pick_split(int N, int K, int sms, bool allow_split, int* kslice) {
    const int nkb = K / 32, tiles = N / 16;
    int ns = 1;
    if (allow_split) {
        ns = max(acb_ceil_div(K, 1536), acb_ceil_div(2 * sms, tiles));
        ns = max(1, min(min(ns, ACB_LM_MAX_SPLIT), nkb / 2 > 0 ? nkb / 2 : 1));
    }
    int kbs = acb_ceil_div(nkb, ns);
    ns = acb_ceil_div(nkb, kbs);   // no empty slices
    *kslice = kbs * 32;
    return ns;
}

// ---- wide GEMM (rows > 64)
static int wide_npad(int rows) { return rows <= 128 ? 128 : 256; }

// K slices of the wide GEMM (grid.y) from (N, K, SM count) alone, never from rows: the count whose CTAs (one per SM: the ring
// takes 144-200 KB) fill the largest share of their waves, up to ACB_LM_MAX_SPLIT `part` slots when the consumer reduces
// partial sums (allow_split), else a cluster of 1, 2 or 4 CTAs.  Sets *kslice (a multiple of WIDE_KC).
static int pick_split_wide(int N, int K, int sms, bool allow_split, int* kslice) {
    const int nch = acb_ceil_div(K, WIDE_KC), tiles = N / 64;
    int best = 1;
    double best_fill = 0.0;
    for (int ns = 1; ns <= (allow_split ? ACB_LM_MAX_SPLIT : 4) && ns <= nch; ns = allow_split ? ns + 1 : 2 * ns) {
        const int ctas = tiles * ns;
        const double fill = (double)ctas / ((double)sms * acb_ceil_div(ctas, sms));
        if (fill > best_fill + 1e-9) { best = ns; best_fill = fill; }
    }
    const int cps = acb_ceil_div(nch, best);   // chunks per slice; no empty slices
    *kslice = cps * WIDE_KC;
    return acb_ceil_div(nch, cps);
}

// grid (N / 64, ny); the non-PARTIAL epilogues run ny as one cluster that reduces the K slices
template <int EPI>
static int launch_wide(const CUtensorMap& wm, const CUtensorMap& xm, int w_row0, const GemmParams& p, int ny, cudaStream_t s,
                       const float* wscale = nullptr) {
    ACB_REQUIRE(p.N % 64 == 0 && p.rows <= 256, "lm_gemm_wide: N=%d rows=%d", p.N, p.rows);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.N / 64, ny);
    cfg.blockDim = dim3(128);
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 1;
    at[0].val.clusterDim.y = EPI == EPI_PARTIAL ? 1 : ny;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    cudaError_t e;
    if (wscale && wide_npad(p.rows) == 128) {
        cfg.dynamicSmemBytes = WideCfg<128, 1>::SMEM;
        e = cudaLaunchKernelEx(&cfg, lm_gemm_wide_fp8_kernel<128, EPI>, wm, xm, p, w_row0, wscale);
    } else if (wscale) {
        cfg.dynamicSmemBytes = WideCfg<256, 1>::SMEM;
        e = cudaLaunchKernelEx(&cfg, lm_gemm_wide_fp8_kernel<256, EPI>, wm, xm, p, w_row0, wscale);
    } else if (wide_npad(p.rows) == 128) {
        cfg.dynamicSmemBytes = WideCfg<128>::SMEM;
        e = cudaLaunchKernelEx(&cfg, lm_gemm_wide_kernel<128, EPI>, wm, xm, p, w_row0);
    } else {
        cfg.dynamicSmemBytes = WideCfg<256>::SMEM;
        e = cudaLaunchKernelEx(&cfg, lm_gemm_wide_kernel<256, EPI>, wm, xm, p, w_row0);
    }
    ACB_CHECK_CUDA(e);
    return ACB_OK;
}

template <int NPAD, int EPI>
static cudaError_t wide_attr_one() {
    cudaError_t e = cudaFuncSetAttribute(lm_gemm_wide_kernel<NPAD, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, WideCfg<NPAD>::SMEM);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(lm_gemm_wide_kernel<NPAD, EPI>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
}
template <int EPI>
static cudaError_t wide_attr_all() {
    cudaError_t e = wide_attr_one<128, EPI>();
    return e != cudaSuccess ? e : wide_attr_one<256, EPI>();
}
template <int NPAD, int EPI>
static cudaError_t wide_fp8_attr_one() {
    cudaError_t e = cudaFuncSetAttribute(lm_gemm_wide_fp8_kernel<NPAD, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         WideCfg<NPAD, 1>::SMEM);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(lm_gemm_wide_fp8_kernel<NPAD, EPI>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
}
template <int EPI>
static cudaError_t wide_fp8_attr_all() {
    cudaError_t e = wide_fp8_attr_one<128, EPI>();
    return e != cudaSuccess ? e : wide_fp8_attr_one<256, EPI>();
}

// Layer l's [N][K] block of a stacked per-layer matrix (fp16 or e4m3 codes) and its row scales (NULL for fp16).
static const void* layer_w(const acb_lm* lm, const void* w, int l, int N, int K) {
    return static_cast<const unsigned char*>(w) + (size_t)l * N * K * (lm->w8 ? 1 : 2);
}
static const float* layer_s(const acb_lm* lm, const float* s, int l, int N) { return lm->w8 ? s + (size_t)l * N : nullptr; }

static GemmParams base_gemm(const void* W, const void* X, int N, int K, int rows, int kslice) {
    GemmParams p{};
    p.W = (const __half*)W;
    p.X = (const __half*)X;
    p.N = N; p.K = K; p.rows = rows; p.kslice = kslice;
    return p;
}


// ACB_DEBUG=1: synchronise and report after every launch of a directly-enqueued step (not during graph capture).
static bool acb_debug_on() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("ACB_DEBUG"); v = (e && e[0] == '1') ? 1 : 0; }
    return v == 1;
}
static int acb_dbg(cudaStream_t s, bool capturing, const char* what, int layer) {
    if (!acb_debug_on() || capturing) return ACB_OK;
    fprintf(stderr, "[acb] %s layer %d ... ", what, layer); fflush(stderr);
    cudaError_t e = cudaStreamSynchronize(s);
    fprintf(stderr, "%s\n", cudaGetErrorString(e)); fflush(stderr);
    if (e != cudaSuccess) { acb_set_error("%s (layer %d): %s", what, layer, cudaGetErrorString(e)); return ACB_ERR_CUDA; }
    return ACB_OK;
}
#define DBG(what, layer) ACB_TRY(acb_dbg(s, capturing, what, layer))

// pf_tokens > 0: PROMPT PREFILL pass (the multi-token first call of the reference, transformer.py:240-247, 413-414, lm.py:513-534):
// the same kernels run on rows * pf_tokens (token, row) pairs -- positions pos .. pos + pf_tokens - 1 of every row at once, causal
// inside the pass because the QKV GEMM appends all of them to the cache before the attention kernel runs -- and stop after the
// last layer (no logits: the next decode step consumes the last prompt position).
// pf_prefix: the pass embeds condition-prefix vectors (lm->prefix) instead of tokens, otherwise it is a prefill pass like any other.
// In an admission (lm->pf_slot >= 0) a pass serves the slot's two rows only: row j of the pass's generation is cache row
// pf_slot + j * slots, and cross attention covers the slot's own text length.
static int pass_rows(const acb_lm* lm) { return lm->pf_slot >= 0 ? 2 : lm->rows; }

static int enqueue_step(acb_lm* lm, cudaStream_t s, float* logits_out, int* n_launch, bool gemms_only = false,
                        bool capturing = false, int pf_tokens = 0, bool pf_prefix = false) {
    const acb_lm_config& c = lm->cfg;
    const acb_lm_buffers& B = lm->buf;
    const bool pf = pf_tokens > 0;
    ACB_REQUIRE(!pf_prefix || (pf && lm->prefix), "enqueue_step: a prefix pass needs the prefix of acb_lm_begin_prefix");
    const bool slot_step = lm->slots && !pf;   // the session's decode step (its passes are an admission's prefix prefill)
    const int rows_real = pf ? pass_rows(lm) : lm->rows, rows = pf ? rows_real * pf_tokens : rows_real;
    const int row0 = pf && lm->pf_slot >= 0 ? lm->pf_slot : 0, row_stride = pf && lm->pf_slot >= 0 ? lm->slots : 1;
    const int text_len = pf && lm->pf_slot >= 0 ? lm->pf_text_len : lm->text_len;
    const int d = c.dim, ffn = c.ffn_dim, L = c.num_layers, H = c.num_heads, nt = nt_for_rows(rows);
    // rows > 64 (then rows_real > 64 and a prefill pass holds one position per row): every GEMM but EPI_CROSSKV on the wide kernel
    const bool wide = rows > 64;
    const size_t part_stride = (size_t)(pf && !wide ? 8 * nt : lm->rows_pad) * d;
    // self-attention cache: a paged session's step reads and appends through the page table (kv_layer: one layer of the
    // pool), its admission's prefix passes run into the staging cache of the slot's two rows (rows 0 and 1), and its prompt
    // passes (paged_pass) write and read the slot's pages through the table
    const bool stage = pf && pf_prefix && lm->paged, paged_pass = pf && !pf_prefix && lm->paged;
    const int kv_len = stage ? lm->max_prefix : c.max_seq, kv_stride = stage ? 1 : row_stride;
    __half* const kv_k = stage ? lm->stage_k : (lm->paged ? lm->pool_k : (__half*)B.k_cache);
    __half* const kv_v = stage ? lm->stage_v : (lm->paged ? lm->pool_v : (__half*)B.v_cache);
    const size_t kv_layer = stage ? (size_t)2 * H * lm->max_prefix * 64
                          : (lm->paged ? (size_t)lm->n_pages * H * ACB_LM_KV_PAGE * 64 : (size_t)c.max_rows * H * c.max_seq * 64);
    const size_t ckv_layer = (size_t)c.max_rows * H * c.max_text * 64;
    const size_t kv_row0 = lm->paged ? 0 : (size_t)row0 * H * c.max_seq * 64, ckv_row0 = (size_t)row0 * H * c.max_text * 64;
    const float scale = 1.0f / sqrtf(64.f);
    // an FP8 pool's layer l: kv_layer codes (bytes) and kv_layer / 64 scales per layer
    auto fp8_layer = [&](int l) {
        return Fp8Pool{(uint8_t*)lm->pool_k + l * kv_layer, (uint8_t*)lm->pool_v + l * kv_layer,
                       lm->pool_ks + l * (kv_layer / 64), lm->pool_vs + l * (kv_layer / 64)};
    };
    int nl = 0, ks = 0;

    if (!gemms_only) {
        const bool sin_pos = c.positional_embedding != 1;
        if (slot_step) lm_embed_slot_kernel<<<rows, 256, 0, s>>>((const __half*)lm->w.emb, lm->w.inv_freq, B.seq, B.slot_state, B.x, d,
                                                                c.n_q, c.card, c.max_seq, lm->slots, c.pos_scale, sin_pos);
        else if (pf && pf_prefix) lm_embed_prefix_kernel<<<rows, 256, 0, s>>>(lm->prefix, lm->w.inv_freq, B.pos, B.x, d, lm->prefix_len,
                                                                       c.pos_scale, rows_real, sin_pos);
        else if (pf && lm->pf_slot >= 0)   // an admission's prompt pass: both rows read the slot's sequence row, as item 0 of a
                                           // generation of batch 1 reads its own
            lm_embed_kernel<true><<<rows, 256, 0, s>>>((const __half*)lm->w.emb, lm->w.inv_freq,
                                                       B.seq + (size_t)lm->pf_slot * c.n_q * c.max_seq, B.pos, B.x, d, c.n_q,
                                                       c.card, c.max_seq, 1, c.pos_scale, rows_real, sin_pos, lm->prefix_len);
        else if (pf) lm_embed_kernel<true><<<rows, 256, 0, s>>>((const __half*)lm->w.emb, lm->w.inv_freq, B.seq, B.pos, B.x, d, c.n_q,
                                                              c.card, c.max_seq, lm->batch, c.pos_scale, rows_real, sin_pos,
                                                              lm->prefix_len);
        else lm_embed_kernel<false><<<rows, 256, 0, s>>>((const __half*)lm->w.emb, lm->w.inv_freq, B.seq, B.pos, B.x, d, c.n_q,
                                                      c.card, c.max_seq, lm->batch, c.pos_scale, rows, sin_pos, lm->prefix_len);
        ACB_LAUNCH_CHECK();
        ++nl;
        DBG("lm_embed_kernel", -1);
    }
    int pending = 0;  // split-K partial sums waiting to be folded into x by the next LN
    auto ln_launch = [&](const float* gamma, const float* beta, int layer) -> int {
        if (gemms_only) return ACB_OK;
        lm_ln_kernel<<<rows, LN_THREADS, 0, s>>>(B.x, B.part, pending, part_stride, gamma, beta, (__half*)B.h16, d);
        ACB_LAUNCH_CHECK();
        ++nl;
        DBG("lm_ln_kernel", layer);
        return ACB_OK;
    };
    auto partial_gemm = [&](const void* W, const float* S, const void* X, int N, int K, int layer, int wm,
                            const CUtensorMap& xm) -> int {
        const int ns = wide ? pick_split_wide(N, K, lm->sms, true, &ks) : pick_split(N, K, lm->sms, true, &ks);
        GemmParams p = base_gemm(layer_w(lm, W, layer, N, K), X, N, K, rows, ks);
        p.out_f32 = B.part; p.ld_out = N; p.split_stride = part_stride;
        const float* ws = layer_s(lm, S, layer, N);
        if (wide) ACB_TRY(launch_wide<EPI_PARTIAL>(lm->wmap[wm], xm, layer * N, p, ns, s, ws));
        else ACB_TRY(launch_gemm<EPI_PARTIAL>(nt, p, ns, s, pick_ft2(N, K, ns, ks, nt, lm->sms), ws));
        ++nl;
        DBG("gemm_EPI_PARTIAL", layer);
        pending = ns;
        return ACB_OK;
    };
    for (int l = 0; l < L; ++l) {
        const float* ln = lm->w.ln + (size_t)l * 6 * d;
        // --- self attention
        ACB_TRY(ln_launch(ln, ln + d, l));
        {
            const int ns = wide ? pick_split_wide(3 * d, d, lm->sms, false, &ks) : pick_split(3 * d, d, lm->sms, false, &ks);
            GemmParams p = base_gemm(layer_w(lm, lm->w.w_qkv, l, 3 * d, d), B.h16, 3 * d, d, rows, ks);
            const float* ws = layer_s(lm, lm->w.s_qkv, l, 3 * d);
            p.q32 = B.q32; p.kc = kv_k + l * kv_layer + kv_row0; p.vc = kv_v + l * kv_layer + kv_row0;
            p.d = d; p.H = H; p.cache_len = kv_len; p.pos = B.pos; p.rows_real = rows_real; p.row_stride = kv_stride;
            p.rope_freq = lm->w.rope_freq; p.pos_scale = c.pos_scale;
            const bool rope = c.positional_embedding != 0;
            const int ft2 = pf ? 1 : pick_ft2(3 * d, d, 1, ks, nt, lm->sms);
            if (slot_step) {   // plain fp32 epilogue into part slot 0 (free between the LN and the out projection), then
                               // the rotary + cache append at each row's own position
                p.out_f32 = B.part; p.ld_out = 3 * d;
                if (wide) ACB_TRY(launch_wide<EPI_F32>(lm->wmap[WM_QKV], lm->xmap_h16, l * 3 * d, p, ns, s, ws));
                else ACB_TRY(launch_gemm<EPI_F32>(nt, p, 1, s, ft2, ws));
                ++nl;
                DBG("gemm_EPI_F32 (qkv)", l);
                if (!gemms_only && lm->fp8) {
                    lm_qkv_slot_paged_fp8_kernel<<<rows, 256, 0, s>>>(B.part, B.slot_state, B.q32, fp8_layer(l), d, H, lm->slots,
                                                                      lm->w.rope_freq, c.pos_scale, rope, lm->page_table,
                                                                      lm->pages_per_row);
                    ACB_LAUNCH_CHECK();
                    ++nl;
                    DBG("lm_qkv_slot_paged_fp8_kernel", l);
                } else if (!gemms_only && lm->paged) {
                    lm_qkv_slot_paged_kernel<<<rows, 256, 0, s>>>(B.part, B.slot_state, B.q32, p.kc, p.vc, d, H, lm->slots,
                                                                  lm->w.rope_freq, c.pos_scale, rope, lm->page_table,
                                                                  lm->pages_per_row);
                    ACB_LAUNCH_CHECK();
                    ++nl;
                    DBG("lm_qkv_slot_paged_kernel", l);
                } else if (!gemms_only) {
                    lm_qkv_slot_kernel<<<rows, 256, 0, s>>>(B.part, B.slot_state, B.q32, p.kc, p.vc, d, H, c.max_seq, lm->slots,
                                                            lm->w.rope_freq, c.pos_scale, rope);
                    ACB_LAUNCH_CHECK();
                    ++nl;
                    DBG("lm_qkv_slot_kernel", l);
                }
            } else if (paged_pass) {   // the pass's plain fp32 epilogue, then the append through the page table
                p.out_f32 = B.part; p.ld_out = 3 * d;
                ACB_TRY(launch_gemm<EPI_F32>(nt, p, 1, s, ft2, ws));
                ++nl;
                DBG("gemm_EPI_F32 (qkv pass)", l);
                if (lm->fp8)
                    lm_qkv_pf_paged_fp8_kernel<<<rows, 256, 0, s>>>(B.part, B.pos, B.q32, fp8_layer(l), d, H, rows_real,
                                                                    lm->w.rope_freq, c.pos_scale, rope, lm->page_table,
                                                                    lm->pages_per_row, row0, row_stride);
                else
                    lm_qkv_pf_paged_kernel<<<rows, 256, 0, s>>>(B.part, B.pos, B.q32, p.kc, p.vc, d, H, rows_real, lm->w.rope_freq,
                                                                c.pos_scale, rope, lm->page_table, lm->pages_per_row, row0,
                                                                row_stride);
                ACB_LAUNCH_CHECK();
                ++nl;
                DBG("lm_qkv_pf_paged_kernel", l);
            } else if (wide) ACB_TRY(rope ? launch_wide<EPI_QKV_ROPE>(lm->wmap[WM_QKV], lm->xmap_h16, l * 3 * d, p, ns, s, ws)
                                   : launch_wide<EPI_QKV>(lm->wmap[WM_QKV], lm->xmap_h16, l * 3 * d, p, ns, s, ws));
            else if (pf) ACB_TRY(rope ? launch_gemm<EPI_QKV_PF_ROPE>(nt, p, 1, s, ft2, ws) : launch_gemm<EPI_QKV_PF>(nt, p, 1, s, ft2, ws));
            else ACB_TRY(rope ? launch_gemm<EPI_QKV_ROPE>(nt, p, 1, s, ft2, ws) : launch_gemm<EPI_QKV>(nt, p, 1, s, ft2, ws));
            if (!slot_step && !paged_pass) {
                ++nl;
                DBG("gemm_EPI_QKV", l);
            }
        }
        if (!gemms_only) {
            AttnParams a{B.q32, 1, 0, kv_k + l * kv_layer + kv_row0, kv_v + l * kv_layer + kv_row0,
                         (__half*)B.a16, H, d, kv_len, B.pos, 0, scale, rows_real, kv_stride};
            if (slot_step && lm->fp8) {
                a.rows_real = lm->slots;
                lm_attn2_slot_paged_fp8_kernel<<<dim3(H, rows), ATT_WARPS * 32, ATT2F8_SMEM, s>>>(a, fp8_layer(l), B.slot_state,
                                                                                                lm->page_table, lm->pages_per_row);
            } else if (slot_step && lm->paged) {
                a.rows_real = lm->slots;
                lm_attn2_slot_paged_kernel<<<dim3(H, rows), ATT_WARPS * 32, ATT2_SMEM, s>>>(a, B.slot_state, lm->page_table,
                                                                                          lm->pages_per_row);
            } else if (slot_step) { a.rows_real = lm->slots; lm_attn2_slot_kernel<<<dim3(H, rows), ATT_WARPS * 32, ATT2_SMEM, s>>>(a, B.slot_state); }
            else if (paged_pass && lm->fp8) lm_attn2_pf_paged_fp8_kernel<<<dim3(H, rows), ATT_WARPS * 32, ATT2F8_SMEM, s>>>(
                    a, fp8_layer(l), lm->page_table, lm->pages_per_row, row0);
            else if (paged_pass) lm_attn2_pf_paged_kernel<<<dim3(H, rows), ATT_WARPS * 32, ATT2_SMEM, s>>>(a, lm->page_table,
                                                                                                      lm->pages_per_row, row0);
            else if (pf) lm_attn2_kernel<true><<<dim3(H, rows), ATT_WARPS * 32, ATT2_SMEM, s>>>(a);
            else lm_attn2_kernel<false><<<dim3(H, rows), ATT_WARPS * 32, ATT2_SMEM, s>>>(a);
            ACB_LAUNCH_CHECK();
            ++nl;
            DBG("lm_attn2_kernel", l);
        }
        ACB_TRY(partial_gemm(lm->w.w_o, lm->w.s_o, B.a16, d, d, l, WM_O, lm->xmap_a16));
        // --- cross attention
        if (lm->has_cross) {
            ACB_TRY(ln_launch(ln + 2 * d, ln + 3 * d, l));
            ACB_TRY(partial_gemm(lm->w.w_cq, lm->w.s_cq, B.h16, d, d, l, WM_CQ, lm->xmap_h16));
            const int nsq = pending;
            pending = 0;   // these partials are the cross-attention queries, not a residual update
            if (!gemms_only) {
                AttnParams a{B.part, nsq, part_stride, (__half*)B.ck_cache + l * ckv_layer + ckv_row0,
                             (__half*)B.cv_cache + l * ckv_layer + ckv_row0, (__half*)B.a16, H, d, c.max_text, B.pos, text_len,
                             scale, rows_real, row_stride};
                if (slot_step) {
                    a.rows_real = lm->slots;
                    lm_cross_attn_slot_kernel<<<acb_ceil_div(rows * H, 8), 256, 0, s>>>(a, rows, B.slot_state);
                } else if (pf) lm_cross_attn_kernel<true><<<acb_ceil_div(rows * H, 8), 256, 0, s>>>(a, rows);
                else lm_cross_attn_kernel<false><<<acb_ceil_div(rows * H, 8), 256, 0, s>>>(a, rows);
                ACB_LAUNCH_CHECK();
                ++nl;
                DBG("lm_cross_attn_kernel", l);
            }
            ACB_TRY(partial_gemm(lm->w.w_co, lm->w.s_co, B.a16, d, d, l, WM_CO, lm->xmap_a16));
        }
        // --- feed forward
        ACB_TRY(ln_launch(ln + 4 * d, ln + 5 * d, l));
        {
            const int ns = wide ? pick_split_wide(ffn, d, lm->sms, false, &ks) : pick_split(ffn, d, lm->sms, false, &ks);
            GemmParams p = base_gemm(layer_w(lm, lm->w.w_ff1, l, ffn, d), B.h16, ffn, d, rows, ks);
            p.out_f16 = (__half*)B.f16; p.ld_out = ffn;
            const float* ws = layer_s(lm, lm->w.s_ff1, l, ffn);
            if (wide) ACB_TRY(launch_wide<EPI_GELU>(lm->wmap[WM_FF1], lm->xmap_h16, l * ffn, p, ns, s, ws));
            else ACB_TRY(launch_gemm<EPI_GELU>(nt, p, 1, s, pick_ft2(ffn, d, 1, ks, nt, lm->sms), ws));
            ++nl;
            DBG("gemm_EPI_GELU", l);
        }
        ACB_TRY(partial_gemm(lm->w.w_ff2, lm->w.s_ff2, B.f16, d, ffn, l, WM_FF2, lm->xmap_f16));
    }
    if (pf) {   // no output norm / heads / sampler: the pass only fills the KV cache
        if (n_launch) *n_launch = nl;
        return ACB_OK;
    }
    ACB_TRY(ln_launch(lm->w.out_norm, lm->w.out_norm + d, -1));
    {
        const int N = c.n_q * c.card;
        const int ns = wide ? pick_split_wide(N, d, lm->sms, false, &ks) : pick_split(N, d, lm->sms, false, &ks);
        GemmParams p = base_gemm(lm->w.heads, B.h16, N, d, rows, ks);
        p.out_f32 = B.logits; p.ld_out = N;
        if (wide) ACB_TRY(launch_wide<EPI_F32>(lm->wmap[WM_HEADS], lm->xmap_h16, 0, p, ns, s));
        else ACB_TRY(launch_gemm<EPI_F32>(nt, p, 1, s, pick_ft2(N, d, 1, ks, nt, lm->sms)));
        ++nl;
        DBG("gemm_EPI_F32", -1);
    }
    if (!gemms_only) {
        int NP = 1;
        while (NP < c.card) NP <<= 1;
        SampleParams sp{B.logits, lm->samp.noise_from_buffer ? B.noise : nullptr, logits_out, B.seq, B.seq_mask, B.pos,
                        c.max_seq, nullptr, lm->batch, rows, c.n_q, c.card, NP, lm->samp.use_sampling, lm->samp.top_k,
                        lm->samp.temp, lm->samp.top_p, lm->samp.cfg_coef, lm->samp.seed, 0, lm->samp.cfg_coef_beta,
                        lm->prefix_len};
        size_t smem = ((size_t)c.card + 2 * (size_t)NP) * sizeof(float);
        if (lm->slots) {
            sp.seq_mask = B.slot_mask; sp.pos = nullptr;
            lm_sample_slot_kernel<<<dim3(c.n_q, lm->slots), 1024, smem, s>>>(sp, B.slot_state, B.slot_sampling);
        } else {
            lm_sample_kernel<<<dim3(c.n_q, lm->batch), 1024, smem, s>>>(sp);
        }
        ACB_LAUNCH_CHECK();
        ++nl;
        DBG("lm_sample_kernel", -1);
    }
    if (n_launch) *n_launch = nl;
    return ACB_OK;
}

extern "C" int acb_lm_create(const acb_lm_config* cfg, const acb_lm_weights* w, const acb_lm_buffers* buf, acb_lm_t** out) {
    ACB_REQUIRE(cfg && w && buf && out, "acb_lm_create: null argument");
    ACB_REQUIRE(cfg->dim % 64 == 0 && cfg->dim == cfg->num_heads * 64, "acb_lm_create: head_dim must be 64 (dim=%d heads=%d)",
                cfg->dim, cfg->num_heads);
    ACB_REQUIRE(cfg->dim <= 4 * LN_THREADS, "acb_lm_create: dim %d too large for the LayerNorm kernel", cfg->dim);
    ACB_REQUIRE(cfg->ffn_dim % 32 == 0 && cfg->card % 16 == 0 && cfg->n_q >= 1 && cfg->n_q <= 16, "acb_lm_create: bad ffn/card/n_q");
    ACB_REQUIRE(cfg->card <= 4096, "acb_lm_create: card %d > 4096 not built", cfg->card);
    ACB_REQUIRE(cfg->max_rows >= 1 && cfg->max_rows <= ACB_LM_MAX_ROWS, "acb_lm_create: max_rows %d not in [1,%d]", cfg->max_rows,
                ACB_LM_MAX_ROWS);
    ACB_REQUIRE(cfg->max_seq >= 2 && cfg->max_seq <= 12000, "acb_lm_create: max_seq %d out of range", cfg->max_seq);
    ACB_REQUIRE(cfg->dim <= 2048, "acb_lm_create: dim %d > 2048: the GEMM stages a 16 x dim weight slab per CTA", cfg->dim);
    ACB_REQUIRE(cfg->positional_embedding >= 0 && cfg->positional_embedding <= 2, "acb_lm_create: positional_embedding %d not in [0,2]",
                cfg->positional_embedding);
    ACB_REQUIRE(cfg->positional_embedding == 0 || w->rope_freq, "acb_lm_create: rotary positions need weights.rope_freq");
    ACB_REQUIRE(cfg->weight_dtype == 0 || cfg->weight_dtype == 1, "acb_lm_create: weight_dtype %d not 0 (fp16) or 1 (e4m3)",
                cfg->weight_dtype);
    ACB_REQUIRE(cfg->weight_dtype == 0 || (w->s_qkv && w->s_o && w->s_ff1 && w->s_ff2 &&
                                           (!cfg->cross_attention || (w->s_cq && w->s_ckv && w->s_co))),
                "acb_lm_create: weight_dtype 1 (e4m3) needs the row scales of every per-layer matrix the model has");
    acb_lm* lm = new (std::nothrow) acb_lm();
    ACB_REQUIRE(lm, "acb_lm_create: out of host memory");
    lm->cfg = *cfg; lm->w = *w; lm->buf = *buf;
    lm->paged = !buf->k_cache && !buf->v_cache;
    lm->w8 = cfg->weight_dtype == 1;
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&lm->sms, cudaDevAttrMultiProcessorCount, dev);
    cudaError_t e = cudaStreamCreateWithFlags(&lm->capture_stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { delete lm; acb_set_error("acb_lm_create: cudaStreamCreate: %s", cudaGetErrorString(e)); return ACB_ERR_CUDA; }
    // every kernel of the step asks for the maximum shared-memory carve-out: the GEMMs stage up to ~70 KB of weights per CTA and
    // the attention ring takes 64 KB, and with one L1 / shared split for all of them an SM never changes its configuration
    // between consecutive kernels of the graph.
    cudaError_t ea = gemm_attr_all<EPI_PARTIAL>();
    if (ea == cudaSuccess) ea = gemm_attr_all<EPI_QKV>();
    if (ea == cudaSuccess) ea = gemm_attr_all<EPI_GELU>();
    if (ea == cudaSuccess) ea = gemm_attr_all<EPI_F32>();
    if (ea == cudaSuccess) ea = gemm_attr_all<EPI_CROSSKV>();
    if (ea == cudaSuccess) ea = gemm_attr_all<EPI_QKV_PF>();
    if (ea == cudaSuccess) ea = gemm_attr_all<EPI_QKV_ROPE>();
    if (ea == cudaSuccess) ea = gemm_attr_all<EPI_QKV_PF_ROPE>();
    if (lm->w8) {
        if (ea == cudaSuccess) ea = gemm_attr_all<EPI_PARTIAL>(true);
        if (ea == cudaSuccess) ea = gemm_attr_all<EPI_QKV>(true);
        if (ea == cudaSuccess) ea = gemm_attr_all<EPI_GELU>(true);
        if (ea == cudaSuccess) ea = gemm_attr_all<EPI_F32>(true);
        if (ea == cudaSuccess) ea = gemm_attr_all<EPI_CROSSKV>(true);
        if (ea == cudaSuccess) ea = gemm_attr_all<EPI_QKV_PF>(true);
        if (ea == cudaSuccess) ea = gemm_attr_all<EPI_QKV_ROPE>(true);
        if (ea == cudaSuccess) ea = gemm_attr_all<EPI_QKV_PF_ROPE>(true);
    }
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT2_SMEM);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT2_SMEM);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_slot_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT2_SMEM);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_slot_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_cross_attn_slot_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_embed_slot_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_qkv_slot_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_slot_paged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT2_SMEM);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_slot_paged_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_qkv_slot_paged_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_pf_paged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT2_SMEM);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_pf_paged_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_slot_paged_fp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT2F8_SMEM);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_slot_paged_fp8_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_qkv_slot_paged_fp8_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_pf_paged_fp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT2F8_SMEM);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_pf_paged_fp8_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_sample_slot_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_cross_attn_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_ln_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_embed_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_embed_prefix_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_sample_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (cfg->max_rows > 64) {
        if (ea == cudaSuccess) ea = wide_attr_all<EPI_PARTIAL>();
        if (ea == cudaSuccess) ea = wide_attr_all<EPI_QKV>();
        if (ea == cudaSuccess) ea = wide_attr_all<EPI_QKV_ROPE>();
        if (ea == cudaSuccess) ea = wide_attr_all<EPI_GELU>();
        if (ea == cudaSuccess) ea = wide_attr_all<EPI_F32>();
        if (lm->w8) {
            if (ea == cudaSuccess) ea = wide_fp8_attr_all<EPI_PARTIAL>();
            if (ea == cudaSuccess) ea = wide_fp8_attr_all<EPI_QKV>();
            if (ea == cudaSuccess) ea = wide_fp8_attr_all<EPI_QKV_ROPE>();
            if (ea == cudaSuccess) ea = wide_fp8_attr_all<EPI_GELU>();
            if (ea == cudaSuccess) ea = wide_fp8_attr_all<EPI_F32>();
        }
    }
    if (ea != cudaSuccess) {
        acb_set_error("acb_lm_create: cudaFuncSetAttribute: %s", cudaGetErrorString(ea));
        cudaStreamDestroy(lm->capture_stream);
        delete lm;
        return ACB_ERR_CUDA;
    }
    if (cfg->max_rows > 64) {   // the wide GEMM's weight maps: each stacked matrix as [L * N][K], 64-row boxes
        const int d = cfg->dim, ffn = cfg->ffn_dim, L = cfg->num_layers;
        auto wmap = lm->w8 ? encode_map_u8 : encode_map;
        int rc = wmap(&lm->wmap[WM_QKV], w->w_qkv, d, L * 3 * d, 64);
        if (rc == ACB_OK) rc = wmap(&lm->wmap[WM_O], w->w_o, d, L * d, 64);
        if (rc == ACB_OK && cfg->cross_attention) rc = wmap(&lm->wmap[WM_CQ], w->w_cq, d, L * d, 64);
        if (rc == ACB_OK && cfg->cross_attention) rc = wmap(&lm->wmap[WM_CO], w->w_co, d, L * d, 64);
        if (rc == ACB_OK) rc = wmap(&lm->wmap[WM_FF1], w->w_ff1, d, L * ffn, 64);
        if (rc == ACB_OK) rc = wmap(&lm->wmap[WM_FF2], w->w_ff2, ffn, L * d, 64);
        if (rc == ACB_OK) rc = encode_map(&lm->wmap[WM_HEADS], w->heads, d, cfg->n_q * cfg->card, 64);
        if (rc != ACB_OK) {
            cudaStreamDestroy(lm->capture_stream);
            delete lm;
            return rc;
        }
    }
    *out = lm;
    return ACB_OK;
}

static void drop_graph(acb_lm* lm) {
    if (lm->exec) { cudaGraphExecDestroy(lm->exec); lm->exec = nullptr; }
    if (lm->graph) { cudaGraphDestroy(lm->graph); lm->graph = nullptr; }
}

extern "C" int acb_lm_destroy(acb_lm_t* lm) {
    if (!lm) return ACB_OK;
    drop_graph(lm);
    if (lm->capture_stream) cudaStreamDestroy(lm->capture_stream);
    delete lm;
    return ACB_OK;
}

__global__ void lm_set_pos_kernel(int* pos, int value) { pos[0] = value; }

// Prefill passes over cache positions [pos0, pos0 + n) of every row, ACB_LM_PREFILL_ROWS / rows positions per pass (one above
// 64 rows: the wide GEMM already shares each weight byte among all rows): token columns pos - prefix_len of buffers.seq, or
// (prefix) the condition-prefix vectors.  Leaves pos = pos0 + n on the device and the padded decode rows [rows, rows_pad) of
// the activation buffers zero.  In an admission (lm->pf_slot >= 0) the passes serve the slot's two rows, so a pass holds
// ACB_LM_PREFILL_ROWS / 2 positions, as in a generation of batch 1 with CFG; the padding restored is the session's.
static int prefill_passes(acb_lm* lm, cudaStream_t s, int pos0, int n, bool prefix) {
    const acb_lm_config& c = lm->cfg;
    const int d = c.dim, rows = pass_rows(lm);
    int per = rows > ACB_LM_PREFILL_ROWS ? 1 : ACB_LM_PREFILL_ROWS / rows;
    // ACB_LM_PREFILL_PER=n: at most n positions per pass (n = 1: one position per pass, the reference order for tests)
    if (const char* e = getenv("ACB_LM_PREFILL_PER")) { const int cap = atoi(e); if (cap >= 1 && cap < per) per = cap; }
    int done = 0;
    while (done < n) {
        const int tc = n - done < per ? n - done : per;
        const int vrows = rows * tc, pad = 8 * nt_for_rows(vrows);
        lm_set_pos_kernel<<<1, 1, 0, s>>>(lm->buf.pos, pos0 + done);
        ACB_LAUNCH_CHECK();
        if (pad > vrows) {   // the GEMMs read their activation rows up to the tile height: rows >= vrows must be zero
            ACB_CHECK_CUDA(cudaMemsetAsync((__half*)lm->buf.h16 + (size_t)vrows * d, 0, (size_t)(pad - vrows) * d * sizeof(__half), s));
            ACB_CHECK_CUDA(cudaMemsetAsync((__half*)lm->buf.a16 + (size_t)vrows * d, 0, (size_t)(pad - vrows) * d * sizeof(__half), s));
            ACB_CHECK_CUDA(cudaMemsetAsync((__half*)lm->buf.f16 + (size_t)vrows * c.ffn_dim, 0, (size_t)(pad - vrows) * c.ffn_dim * sizeof(__half), s));
        }
        ACB_TRY(enqueue_step(lm, s, nullptr, nullptr, false, false, tc, prefix));
        done += tc;
    }
    lm_set_pos_kernel<<<1, 1, 0, s>>>(lm->buf.pos, pos0 + n);
    ACB_LAUNCH_CHECK();
    // back to decode: its padded rows [rows, rows_pad) must be zero again
    if (lm->rows_pad > lm->rows) {
        ACB_CHECK_CUDA(cudaMemsetAsync((__half*)lm->buf.h16 + (size_t)lm->rows * d, 0, (size_t)(lm->rows_pad - lm->rows) * d * sizeof(__half), s));
        ACB_CHECK_CUDA(cudaMemsetAsync((__half*)lm->buf.a16 + (size_t)lm->rows * d, 0, (size_t)(lm->rows_pad - lm->rows) * d * sizeof(__half), s));
        ACB_CHECK_CUDA(cudaMemsetAsync((__half*)lm->buf.f16 + (size_t)lm->rows * c.ffn_dim, 0, (size_t)(lm->rows_pad - lm->rows) * c.ffn_dim * sizeof(__half), s));
    }
    return ACB_OK;
}

// Capture one decode step; its kernels are chained by plain stream-order edges.  (Launched with programmatic dependent launch,
// the same kernels gave wrong logits on the H100 once the KV cache held more than a few positions, for a cause not found.)
static int capture_step(acb_lm* lm) {
    drop_graph(lm);
    ACB_CHECK_CUDA(cudaStreamBeginCapture(lm->capture_stream, cudaStreamCaptureModeThreadLocal));
    int rc = enqueue_step(lm, lm->capture_stream, nullptr, &lm->launches, false, true);
    cudaError_t e = cudaStreamEndCapture(lm->capture_stream, &lm->graph);
    if (rc == ACB_OK && e == cudaSuccess) e = cudaGraphInstantiate(&lm->exec, lm->graph, 0);
    if (rc == ACB_OK && e == cudaSuccess) return ACB_OK;
    cudaGetLastError();
    drop_graph(lm);
    if (rc == ACB_OK) acb_set_error("acb_lm_begin: graph capture failed: %s", cudaGetErrorString(e));
    return rc != ACB_OK ? rc : ACB_ERR_CUDA;
}

extern "C" int acb_lm_begin(acb_lm_t* lm, const float* cross, int batch, int rows, int text_len, int seq_len,
                            const acb_lm_sampling* sampling, void* stream) {
    return acb_lm_begin_prefix(lm, cross, nullptr, 0, batch, rows, text_len, seq_len, sampling, stream);
}

extern "C" int acb_lm_begin_prefix(acb_lm_t* lm, const float* cross, const float* prefix, int prefix_len, int batch, int rows,
                                   int text_len, int seq_len, const acb_lm_sampling* sampling, void* stream) {
    ACB_REQUIRE(lm && sampling, "acb_lm_begin: null argument");
    ACB_REQUIRE(!lm->paged, "acb_lm_begin: the handle has no contiguous KV cache (buffers.k_cache is NULL: a paged handle)");
    const acb_lm_config& c = lm->cfg;
    ACB_REQUIRE(batch >= 1 && (rows == batch || rows == 2 * batch || rows == 3 * batch), "acb_lm_begin: rows must be batch, 2*batch (CFG) or 3*batch (double CFG)");
    ACB_REQUIRE(rows <= c.max_rows, "acb_lm_begin: rows %d > max_rows %d", rows, c.max_rows);
    ACB_REQUIRE(prefix_len >= 0 && (prefix_len == 0 || prefix), "acb_lm_begin: prefix_len %d without a prefix tensor", prefix_len);
    ACB_REQUIRE(seq_len >= 2 && prefix_len + seq_len <= c.max_seq, "acb_lm_begin: prefix %d + seq_len %d > max_seq %d", prefix_len,
                seq_len, c.max_seq);
    if (rows > 64 && (c.ffn_dim % 64 != 0 || (c.n_q * c.card) % 64 != 0)) {
        acb_set_error("acb_lm_begin: rows %d > 64 run the wide GEMM, which needs ffn_dim (%d) and n_q * card (%d) to be multiples of 64",
                      rows, c.ffn_dim, c.n_q * c.card);
        return ACB_ERR_UNSUPPORTED;
    }
    ACB_REQUIRE(!c.cross_attention || cross, "acb_lm_begin: the model has cross attention, a condition tensor is required"
                " (the reference asserts the same, transformer.py:553-556)");
    ACB_REQUIRE(!cross || (text_len >= 1 && text_len <= c.max_text), "acb_lm_begin: text_len %d out of range", text_len);
    lm->slots = 0;
    cudaStream_t s = (cudaStream_t)stream;
    const int d = c.dim, H = c.num_heads;
    if (rows > 64) {   // the wide GEMM's activation maps: rows past `rows` of a box are zero-filled
        const int npad = wide_npad(rows);
        ACB_TRY(encode_map(&lm->xmap_h16, lm->buf.h16, d, rows, npad));
        ACB_TRY(encode_map(&lm->xmap_a16, lm->buf.a16, d, rows, npad));
        ACB_TRY(encode_map(&lm->xmap_f16, lm->buf.f16, c.ffn_dim, rows, npad));
    }
    lm->batch = batch; lm->rows = rows; lm->rows_pad = rows > 64 ? wide_npad(rows) : 8 * nt_for_rows(rows); lm->text_len = text_len; lm->seq_len = seq_len;
    lm->prefix_len = prefix_len; lm->prefix = prefix;
    lm->samp = *sampling;
    lm->has_cross = c.cross_attention && cross;
    // zero the padded activation rows once; kernels only ever write rows < `rows`
    ACB_CHECK_CUDA(cudaMemsetAsync(lm->buf.h16, 0, (size_t)lm->rows_pad * d * sizeof(__half), s));
    ACB_CHECK_CUDA(cudaMemsetAsync(lm->buf.a16, 0, (size_t)lm->rows_pad * d * sizeof(__half), s));
    ACB_CHECK_CUDA(cudaMemsetAsync(lm->buf.f16, 0, (size_t)lm->rows_pad * c.ffn_dim * sizeof(__half), s));
    int hp[4] = {0, 0, batch, text_len};   // pos, finished-block counter of the sampler, (info) batch, text_len
    ACB_CHECK_CUDA(cudaMemcpyAsync(lm->buf.pos, hp, sizeof(hp), cudaMemcpyHostToDevice, s));
    if (lm->has_cross) {
        const size_t M = (size_t)rows * text_len, Mpad = (M + 63) / 64 * 64;
        lm_f32_to_f16_kernel<<<(unsigned)((Mpad * d + 255) / 256), 256, 0, s>>>(cross, (__half*)lm->buf.cross16, M * d, Mpad * d);
        ACB_LAUNCH_CHECK();
        const size_t ckv_layer = (size_t)c.max_rows * H * c.max_text * 64;
        for (int l = 0; l < c.num_layers; ++l)
            for (size_t r0 = 0; r0 < M; r0 += 64) {
                int ks = 0;
                pick_split(2 * d, d, lm->sms, false, &ks);
                GemmParams p = base_gemm(layer_w(lm, lm->w.w_ckv, l, 2 * d, d),
                                         (const __half*)lm->buf.cross16 + r0 * d, 2 * d, d, (int)min((size_t)64, M - r0), ks);
                p.kc = (__half*)lm->buf.ck_cache + l * ckv_layer; p.vc = (__half*)lm->buf.cv_cache + l * ckv_layer;
                p.d = d; p.H = H; p.cache_len = c.max_text; p.text_len = text_len; p.row0 = (int)r0;
                ACB_TRY(launch_gemm<EPI_CROSSKV>(8, p, 1, s, 1, layer_s(lm, lm->w.s_ckv, l, 2 * d)));
            }
    }
    // the condition prefix fills cache positions [0, prefix_len) once per generate (after the cross K/V: the passes attend to
    // them); decode and prompt prefill then run at cache position prefix_len + sequence column
    if (prefix_len > 0) ACB_TRY(prefill_passes(lm, s, 0, prefix_len, true));
    lm->prefix = nullptr;   // read only by the passes just enqueued: the caller's tensor is not referenced after this call
    // opt in to large dynamic shared memory where needed
    {
        int NP = 1;
        while (NP < c.card) NP <<= 1;
        size_t smem = ((size_t)c.card + 2 * (size_t)NP) * sizeof(float);
        if (smem > 48 * 1024)
            ACB_CHECK_CUDA(cudaFuncSetAttribute(lm_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    return capture_step(lm);
}

// Prompt prefill: consume sequence columns [pos0, pos0 + n_tokens) of every row (their tokens are already in buffers.seq)
// without sampling, ACB_LM_PREFILL_ROWS / rows positions per pass, at cache positions prefix_len + column.  Leaves
// pos = prefix_len + pos0 + n_tokens on the device.
extern "C" int acb_lm_prefill(acb_lm_t* lm, int pos0, int n_tokens, void* stream) {
    ACB_REQUIRE(lm && lm->rows > 0, "acb_lm_prefill: call acb_lm_begin first");
    ACB_REQUIRE(!lm->paged, "acb_lm_prefill: the handle has no contiguous KV cache (a paged handle)");
    ACB_REQUIRE(!lm->slots, "acb_lm_prefill: a slot session consumes prompts one column per step");
    ACB_REQUIRE(pos0 >= 0 && n_tokens >= 0 && pos0 + n_tokens < lm->seq_len, "acb_lm_prefill: positions [%d, %d) exceed the sequence (%d)",
                pos0, pos0 + n_tokens, lm->seq_len);
    return prefill_passes(lm, (cudaStream_t)stream, lm->prefix_len + pos0, n_tokens, false);
}

// ------------------------------------------------------------------------------------------------ slot mode
// The session set-up shared by acb_lm_begin_slots and acb_lm_begin_slots_paged (which sets the pool fields first).
static int begin_slots(acb_lm_t* lm, int slots, int max_text, int seq_len_max, const acb_lm_sampling* sampling, void* stream) {
    const acb_lm_config& c = lm->cfg;
    ACB_REQUIRE(lm->buf.slot_sampling && lm->buf.slot_state && lm->buf.slot_mask,
                "acb_lm_begin_slots: buffers.slot_sampling, slot_state and slot_mask are required");
    ACB_REQUIRE(slots >= 1 && slots <= ACB_LM_MAX_SLOTS && 2 * slots <= c.max_rows, "acb_lm_begin_slots: slots %d not in [1, %d] "
                "or 2 * slots > max_rows %d", slots, ACB_LM_MAX_SLOTS, c.max_rows);
    ACB_REQUIRE(seq_len_max >= 2 && seq_len_max <= c.max_seq, "acb_lm_begin_slots: seq_len_max %d not in [2, max_seq %d]",
                seq_len_max, c.max_seq);
    ACB_REQUIRE(!c.cross_attention || (max_text >= 1 && max_text <= c.max_text), "acb_lm_begin_slots: max_text %d not in [1, %d]",
                max_text, c.max_text);
    if (sampling->cfg_coef_beta != 0.f) {
        acb_set_error("acb_lm_begin_slots: double CFG (cfg_coef_beta) is not built in slot mode: a session is [cond; null] rows");
        return ACB_ERR_UNSUPPORTED;
    }
    ACB_REQUIRE(!sampling->noise_from_buffer, "acb_lm_begin_slots: slot mode samples with the on-device Philox noise only");
    const int rows = 2 * slots;
    if (rows > 64 && (c.ffn_dim % 64 != 0 || (c.n_q * c.card) % 64 != 0)) {
        acb_set_error("acb_lm_begin_slots: rows %d > 64 run the wide GEMM, which needs ffn_dim (%d) and n_q * card (%d) to be "
                      "multiples of 64", rows, c.ffn_dim, c.n_q * c.card);
        return ACB_ERR_UNSUPPORTED;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int d = c.dim;
    if (rows > 64) {
        const int npad = wide_npad(rows);
        ACB_TRY(encode_map(&lm->xmap_h16, lm->buf.h16, d, rows, npad));
        ACB_TRY(encode_map(&lm->xmap_a16, lm->buf.a16, d, rows, npad));
        ACB_TRY(encode_map(&lm->xmap_f16, lm->buf.f16, c.ffn_dim, rows, npad));
    }
    lm->slots = slots; lm->batch = slots; lm->rows = rows;
    lm->rows_pad = rows > 64 ? wide_npad(rows) : 8 * nt_for_rows(rows);
    lm->text_len = max_text; lm->seq_len = seq_len_max; lm->prefix_len = 0; lm->prefix = nullptr;
    lm->samp = *sampling;
    lm->has_cross = c.cross_attention != 0;
    ACB_CHECK_CUDA(cudaMemsetAsync(lm->buf.h16, 0, (size_t)lm->rows_pad * d * sizeof(__half), s));
    ACB_CHECK_CUDA(cudaMemsetAsync(lm->buf.a16, 0, (size_t)lm->rows_pad * d * sizeof(__half), s));
    ACB_CHECK_CUDA(cudaMemsetAsync(lm->buf.f16, 0, (size_t)lm->rows_pad * c.ffn_dim * sizeof(__half), s));
    ACB_CHECK_CUDA(cudaMemsetAsync(lm->buf.slot_state, 0, (size_t)slots * ACB_LM_SLOT_STRIDE * sizeof(int), s));   // all INACTIVE
    int NP = 1;
    while (NP < c.card) NP <<= 1;
    const size_t smem = ((size_t)c.card + 2 * (size_t)NP) * sizeof(float);
    if (smem > 48 * 1024)
        ACB_CHECK_CUDA(cudaFuncSetAttribute(lm_sample_slot_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    return capture_step(lm);
}

extern "C" int acb_lm_begin_slots(acb_lm_t* lm, int slots, int max_text, int seq_len_max, const acb_lm_sampling* sampling,
                                  void* stream) {
    ACB_REQUIRE(lm && sampling, "acb_lm_begin_slots: null argument");
    ACB_REQUIRE(!lm->paged, "acb_lm_begin_slots: the handle has no contiguous KV cache (a paged handle: acb_lm_begin_slots_paged)");
    return begin_slots(lm, slots, max_text, seq_len_max, sampling, stream);
}

// acb_lm_begin_slots_paged (k_scale = v_scale = NULL: an fp16 pool) and acb_lm_begin_slots_paged_fp8.
static int begin_slots_paged(acb_lm_t* lm, int slots, int max_text, int seq_len_max, int max_prefix, void* k_pool, void* v_pool,
                             float* k_scale, float* v_scale, int n_pages, int32_t* page_table, int pages_per_row, void* stage_k,
                             void* stage_v, const acb_lm_sampling* sampling, void* stream) {
    ACB_REQUIRE(lm && sampling && k_pool && v_pool && page_table, "acb_lm_begin_slots_paged: null argument");
    ACB_REQUIRE(lm->paged, "acb_lm_begin_slots_paged: the handle was created with a contiguous KV cache (buffers.k_cache)");
    const acb_lm_config& c = lm->cfg;
    ACB_REQUIRE(max_prefix >= 0 && seq_len_max >= 2 && max_prefix + seq_len_max <= c.max_seq,
                "acb_lm_begin_slots_paged: max_prefix %d + seq_len_max %d not in [2, max_seq %d]", max_prefix, seq_len_max, c.max_seq);
    ACB_REQUIRE(max_prefix == 0 || (stage_k && stage_v), "acb_lm_begin_slots_paged: max_prefix > 0 needs the staging buffers");
    const int need = acb_ceil_div(max_prefix + seq_len_max, ACB_LM_KV_PAGE);
    ACB_REQUIRE(pages_per_row >= need && pages_per_row <= ACB_LM_MAX_PAGES_PER_ROW,
                "acb_lm_begin_slots_paged: pages_per_row %d not in [%d, %d]", pages_per_row, need, ACB_LM_MAX_PAGES_PER_ROW);
    ACB_REQUIRE(n_pages >= 2 * need, "acb_lm_begin_slots_paged: %d pages cannot hold one request of %d positions (%d pages)",
                n_pages, max_prefix + seq_len_max, 2 * need);
    lm->pool_k = (__half*)k_pool; lm->pool_v = (__half*)v_pool; lm->n_pages = n_pages;
    lm->page_table = page_table; lm->pages_per_row = pages_per_row;
    lm->stage_k = (__half*)stage_k; lm->stage_v = (__half*)stage_v; lm->max_prefix = max_prefix;
    lm->fp8 = k_scale != nullptr; lm->pool_ks = k_scale; lm->pool_vs = v_scale;
    return begin_slots(lm, slots, max_text, seq_len_max, sampling, stream);
}

extern "C" int acb_lm_begin_slots_paged(acb_lm_t* lm, int slots, int max_text, int seq_len_max, int max_prefix, void* k_pool,
                                        void* v_pool, int n_pages, int32_t* page_table, int pages_per_row, void* stage_k,
                                        void* stage_v, const acb_lm_sampling* sampling, void* stream) {
    return begin_slots_paged(lm, slots, max_text, seq_len_max, max_prefix, k_pool, v_pool, nullptr, nullptr, n_pages, page_table,
                             pages_per_row, stage_k, stage_v, sampling, stream);
}

extern "C" int acb_lm_begin_slots_paged_fp8(acb_lm_t* lm, int slots, int max_text, int seq_len_max, int max_prefix,
                                            void* k_pool, void* v_pool, float* k_scale, float* v_scale, int n_pages,
                                            int32_t* page_table, int pages_per_row, void* stage_k, void* stage_v,
                                            const acb_lm_sampling* sampling, void* stream) {
    ACB_REQUIRE(k_scale && v_scale, "acb_lm_begin_slots_paged_fp8: null scale pool");
    return begin_slots_paged(lm, slots, max_text, seq_len_max, max_prefix, k_pool, v_pool, k_scale, v_scale, n_pages, page_table,
                             pages_per_row, stage_k, stage_v, sampling, stream);
}

extern "C" int acb_lm_admit(acb_lm_t* lm, int slot, const float* cross, int text_len, int seq_len, uint64_t seed,
                            const acb_lm_sampling* sampling, void* stream) {
    return acb_lm_admit_prefix(lm, slot, cross, text_len, nullptr, 0, seq_len, seed, sampling, stream);
}

// acb_lm_admit_prefix, acb_lm_admit_paged and acb_lm_admit_prompt: pages is NULL in a contiguous session, n_page_ids its
// length otherwise; prefill_cols sequence columns are prefilled after the prefix and the slot starts at that column.
static int admit(acb_lm_t* lm, int slot, const float* cross, int text_len, const float* prefix, int prefix_len, int seq_len,
                 int prefill_cols, uint64_t seed, const acb_lm_sampling* sampling, const int32_t* pages, int n_page_ids,
                 void* stream) {
    ACB_REQUIRE(lm && lm->slots > 0, "acb_lm_admit: call acb_lm_begin_slots first");
    ACB_REQUIRE(lm->paged == (pages != nullptr), "%s", lm->paged ? "acb_lm_admit: a paged session admits with acb_lm_admit_paged"
                                                                 : "acb_lm_admit_paged: the session is not paged");
    const acb_lm_config& c = lm->cfg;
    ACB_REQUIRE(slot >= 0 && slot < lm->slots, "acb_lm_admit: slot %d not in [0, %d)", slot, lm->slots);
    ACB_REQUIRE(seq_len >= 2 && seq_len <= lm->seq_len, "acb_lm_admit: seq_len %d not in [2, %d]", seq_len, lm->seq_len);
    ACB_REQUIRE(prefix_len >= 0 && (prefix_len == 0 || prefix), "acb_lm_admit: prefix_len %d without a prefix tensor", prefix_len);
    ACB_REQUIRE(prefix_len + seq_len <= c.max_seq, "acb_lm_admit: prefix %d + seq_len %d > max_seq %d", prefix_len, seq_len,
                c.max_seq);
    ACB_REQUIRE(prefill_cols >= 0 && prefill_cols <= seq_len - 2, "acb_lm_admit_prompt: prefill_cols %d not in [0, seq_len - 2 = %d]",
                prefill_cols, seq_len - 2);
    ACB_REQUIRE(!lm->has_cross || (cross && text_len >= 1 && text_len <= lm->text_len),
                "acb_lm_admit: the model has cross attention: a condition of 1 .. %d text positions is required (got %d)",
                lm->text_len, text_len);
    if (sampling) {
        if (sampling->cfg_coef_beta != 0.f) {
            acb_set_error("acb_lm_admit: double CFG (cfg_coef_beta) is not built in slot mode: a session is [cond; null] rows");
            return ACB_ERR_UNSUPPORTED;
        }
        ACB_REQUIRE(!sampling->noise_from_buffer, "acb_lm_admit: slot mode samples with the on-device Philox noise only");
        ACB_REQUIRE(sampling->temp >= 0.f && sampling->top_k >= 0 && sampling->top_p >= 0.f && sampling->top_p <= 1.f &&
                    isfinite(sampling->temp) && isfinite(sampling->cfg_coef),
                    "acb_lm_admit: needs 0 <= temp < inf (got %g), top_k >= 0 (got %d), 0 <= top_p <= 1 (got %g) and a finite "
                    "cfg_coef (got %g)", sampling->temp, sampling->top_k, sampling->top_p, sampling->cfg_coef);
    }
    PageList pl;
    const int ppr = lm->paged ? acb_ceil_div(prefix_len + seq_len, ACB_LM_KV_PAGE) : 0;
    if (lm->paged) {   // every check before anything is enqueued
        ACB_REQUIRE(prefix_len <= lm->max_prefix, "acb_lm_admit_paged: prefix_len %d > the session's max_prefix %d", prefix_len,
                    lm->max_prefix);
        ACB_REQUIRE(n_page_ids == 2 * ppr && ppr <= lm->pages_per_row, "acb_lm_admit_paged: %d page ids for %d positions: needs "
                    "2 x %d", n_page_ids, prefix_len + seq_len, ppr);
        std::vector<uint8_t> seen((size_t)lm->n_pages, 0);
        for (int i = 0; i < n_page_ids; ++i) {
            const int id = pages[i];
            ACB_REQUIRE(id >= 0 && id < lm->n_pages, "acb_lm_admit_paged: page id %d not in [0, %d)", id, lm->n_pages);
            ACB_REQUIRE(!seen[id], "acb_lm_admit_paged: page %d given twice", id);
            seen[id] = 1;
            pl.ids[i] = id;
        }
    }
    const acb_lm_sampling& sp = sampling ? *sampling : lm->samp;
    cudaStream_t s = (cudaStream_t)stream;
    if (lm->paged) {
        lm_page_table_kernel<<<1, 256, 0, s>>>(lm->page_table, lm->pages_per_row, slot, lm->slots + slot, ppr, pl);
        ACB_LAUNCH_CHECK();
    }
    if (lm->has_cross) {
        // cross K/V of the slot's cond row (slot) and null row (slots + slot), each staged and projected on its own: the
        // EPI_CROSSKV epilogue writes cache row R / text_len = 0 of the destination pointer
        const int d = c.dim, H = c.num_heads;
        const size_t ckv_layer = (size_t)c.max_rows * H * c.max_text * 64, row_elems = (size_t)H * c.max_text * 64;
        const size_t M = (size_t)text_len, Mpad = (M + 63) / 64 * 64;
        for (int half = 0; half < 2; ++half) {
            const int dst = half ? lm->slots + slot : slot;
            lm_f32_to_f16_kernel<<<(unsigned)((Mpad * d + 255) / 256), 256, 0, s>>>(cross + (size_t)half * M * d,
                                                                                   (__half*)lm->buf.cross16, M * d, Mpad * d);
            ACB_LAUNCH_CHECK();
            for (int l = 0; l < c.num_layers; ++l)
                for (size_t r0 = 0; r0 < M; r0 += 64) {
                    int ks = 0;
                    pick_split(2 * d, d, lm->sms, false, &ks);
                    GemmParams p = base_gemm(layer_w(lm, lm->w.w_ckv, l, 2 * d, d),
                                             (const __half*)lm->buf.cross16 + r0 * d, 2 * d, d, (int)min((size_t)64, M - r0), ks);
                    p.kc = (__half*)lm->buf.ck_cache + l * ckv_layer + dst * row_elems;
                    p.vc = (__half*)lm->buf.cv_cache + l * ckv_layer + dst * row_elems;
                    p.d = d; p.H = H; p.cache_len = c.max_text; p.text_len = text_len; p.row0 = (int)r0;
                    ACB_TRY(launch_gemm<EPI_CROSSKV>(8, p, 1, s, 1, layer_s(lm, lm->w.s_ckv, l, 2 * d)));
                }
        }
    }
    // the condition prefix fills cache positions [0, prefix_len) of the slot's two rows (after the cross K/V: the passes attend
    // to them), in the passes acb_lm_begin_prefix runs for a generation of batch 1, so the K/V are the ones it writes.  The
    // passes use the activation buffers and buffers.pos, which the session's step does not carry from one step to the next.
    if (prefix_len > 0) {
        lm->pf_slot = slot; lm->pf_text_len = lm->has_cross ? text_len : 0;
        lm->prefix = prefix; lm->prefix_len = prefix_len;
        const int rc = prefill_passes(lm, s, 0, prefix_len, true);
        lm->pf_slot = -1; lm->pf_text_len = 0;
        lm->prefix = nullptr; lm->prefix_len = 0;   // the session's step reads column = position (its sampler's seq_off is 0)
        ACB_TRY(rc);
        if (lm->fp8) {   // the passes ran into the fp16 staging cache: quantize it into the slot's pages
            const size_t n_vec = (size_t)c.num_layers * 2 * c.num_heads * prefix_len * 2;
            lm_prefix_scatter_fp8_kernel<<<(unsigned)((n_vec * 32 + 255) / 256), 256, 0, s>>>(
                lm->stage_k, lm->stage_v, Fp8Pool{(uint8_t*)lm->pool_k, (uint8_t*)lm->pool_v, lm->pool_ks, lm->pool_vs},
                lm->page_table, lm->pages_per_row, slot, lm->slots + slot, c.num_heads, lm->max_prefix, prefix_len,
                (size_t)lm->n_pages * c.num_heads * ACB_LM_KV_PAGE, n_vec);
            ACB_LAUNCH_CHECK();
        } else if (lm->paged) {   // the passes ran into the staging cache: copy it into the slot's pages
            const size_t total = (size_t)c.num_layers * 2 * c.num_heads * prefix_len * 8;
            lm_prefix_scatter_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
                lm->stage_k, lm->stage_v, lm->pool_k, lm->pool_v, lm->page_table, lm->pages_per_row, slot, lm->slots + slot,
                c.num_heads, lm->max_prefix, prefix_len, (size_t)lm->n_pages * c.num_heads * ACB_LM_KV_PAGE * 64, total);
            ACB_LAUNCH_CHECK();
        }
    }
    // the prompt's columns [0, prefill_cols) at cache positions prefix_len + column, after the prefix (they attend to it), in
    // the passes acb_lm_prefill runs for a generation of batch 1 with CFG.  Both rows embed the slot's sequence row; a paged
    // session's passes append to and attend through the slot's pages (lm_qkv_pf_paged_kernel, lm_attn2_pf_paged_kernel).
    if (prefill_cols > 0) {
        lm->pf_slot = slot; lm->pf_text_len = lm->has_cross ? text_len : 0;
        lm->prefix = nullptr; lm->prefix_len = prefix_len;
        const int rc = prefill_passes(lm, s, prefix_len, prefill_cols, false);
        lm->pf_slot = -1; lm->pf_text_len = 0;
        lm->prefix_len = 0;
        ACB_TRY(rc);
    }
    lm_slot_sampling_kernel<<<1, 1, 0, s>>>(lm->buf.slot_sampling, slot, sp.use_sampling, sp.temp, sp.top_k, sp.top_p,
                                            sp.cfg_coef);
    ACB_LAUNCH_CHECK();
    lm_slot_admit_kernel<<<1, 1, 0, s>>>(lm->buf.slot_state, slot, seq_len, lm->has_cross ? text_len : 0, prefix_len,
                                         (uint32_t)seed, (uint32_t)(seed >> 32));
    ACB_LAUNCH_CHECK();
    if (prefill_cols > 0) {   // the slot starts at column prefill_cols (the admission kernel starts it at 0)
        lm_set_pos_kernel<<<1, 1, 0, s>>>(lm->buf.slot_state + (size_t)slot * ACB_LM_SLOT_STRIDE + ACB_SLOT_POS, prefill_cols);
        ACB_LAUNCH_CHECK();
    }
    return ACB_OK;
}

extern "C" int acb_lm_admit_prefix(acb_lm_t* lm, int slot, const float* cross, int text_len, const float* prefix, int prefix_len,
                                   int seq_len, uint64_t seed, const acb_lm_sampling* sampling, void* stream) {
    return admit(lm, slot, cross, text_len, prefix, prefix_len, seq_len, 0, seed, sampling, nullptr, 0, stream);
}

extern "C" int acb_lm_admit_paged(acb_lm_t* lm, int slot, const float* cross, int text_len, const float* prefix, int prefix_len,
                                  int seq_len, uint64_t seed, const acb_lm_sampling* sampling, const int32_t* pages, int n,
                                  void* stream) {
    ACB_REQUIRE(pages, "acb_lm_admit_paged: null page list");
    return admit(lm, slot, cross, text_len, prefix, prefix_len, seq_len, 0, seed, sampling, pages, n, stream);
}

extern "C" int acb_lm_admit_prompt(acb_lm_t* lm, int slot, const float* cross, int text_len, const float* prefix, int prefix_len,
                                   int seq_len, int prefill_cols, uint64_t seed, const acb_lm_sampling* sampling,
                                   const int32_t* pages, int n_page_ids, void* stream) {
    return admit(lm, slot, cross, text_len, prefix, prefix_len, seq_len, prefill_cols, seed, sampling, pages, n_page_ids, stream);
}

extern "C" int acb_lm_retire(acb_lm_t* lm, int slot, void* stream) {
    ACB_REQUIRE(lm && lm->slots > 0, "acb_lm_retire: call acb_lm_begin_slots first");
    ACB_REQUIRE(slot >= 0 && slot < lm->slots, "acb_lm_retire: slot %d not in [0, %d)", slot, lm->slots);
    lm_slot_retire_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(lm->buf.slot_state, slot);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

extern "C" int acb_lm_slot_status(acb_lm_t* lm, int* out, void* stream) {
    ACB_REQUIRE(lm && lm->slots > 0 && out, "acb_lm_slot_status: call acb_lm_begin_slots first");
    ACB_CHECK_CUDA(cudaMemcpy2DAsync(out, 2 * sizeof(int), lm->buf.slot_state, ACB_LM_SLOT_STRIDE * sizeof(int), 2 * sizeof(int),
                                     lm->slots, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return ACB_OK;
}

extern "C" int acb_lm_uses_pdl(const acb_lm_t*) { return 0; }

extern "C" int acb_lm_steps(acb_lm_t* lm, int n_steps, void* stream) {
    ACB_REQUIRE(lm && lm->exec, "acb_lm_steps: call acb_lm_begin first");
    ACB_REQUIRE(n_steps >= 0, "acb_lm_steps: negative step count");
    for (int i = 0; i < n_steps; ++i) ACB_CHECK_CUDA(cudaGraphLaunch(lm->exec, (cudaStream_t)stream));
    return ACB_OK;
}

extern "C" int acb_lm_step_logits(acb_lm_t* lm, float* logits_out, void* stream) {
    ACB_REQUIRE(lm && lm->rows > 0, "acb_lm_step_logits: call acb_lm_begin first");
    return enqueue_step(lm, (cudaStream_t)stream, logits_out, nullptr);
}

extern "C" int acb_lm_debug_gemms(acb_lm_t* lm, void* stream, int* n_launches) {
    ACB_REQUIRE(lm && lm->rows > 0, "acb_lm_debug_gemms: call acb_lm_begin first");
    return enqueue_step(lm, (cudaStream_t)stream, nullptr, n_launches, true);
}

extern "C" int acb_lm_rows_pad(int rows) {
    ACB_REQUIRE(rows <= ACB_LM_MAX_ROWS, "acb_lm_rows_pad: rows %d > %d", rows, ACB_LM_MAX_ROWS);
    if (rows > 64) return wide_npad(rows);
    return rows <= 16 ? 16 : 8 * nt_for_rows(rows);
}

extern "C" int acb_lm_launches_per_step(const acb_lm_t* lm) { return lm ? lm->launches : 0; }

extern "C" int acb_sample(const float* logits, const float* noise, int64_t* tokens, int batch, int rows, int n_q, int card,
                          const acb_lm_sampling* sampling, uint64_t step, void* stream) {
    ACB_REQUIRE(logits && tokens && sampling, "acb_sample: null argument");
    ACB_REQUIRE(batch >= 1 && (rows == batch || rows == 2 * batch || rows == 3 * batch) && n_q >= 1 && card >= 2 && card <= 4096, "acb_sample: bad shape");
    int NP = 1;
    while (NP < card) NP <<= 1;
    SampleParams sp{logits, sampling->noise_from_buffer ? noise : nullptr, nullptr, nullptr, nullptr, nullptr, 0, tokens, batch, rows, n_q, card, NP,
                    sampling->use_sampling, sampling->top_k, sampling->temp, sampling->top_p, sampling->cfg_coef,
                    sampling->seed, (uint32_t)step, sampling->cfg_coef_beta, 0};
    size_t smem = ((size_t)card + 2 * (size_t)NP) * sizeof(float);
    if (smem > 48 * 1024)
        ACB_CHECK_CUDA(cudaFuncSetAttribute(lm_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    lm_sample_kernel<<<dim3(n_q, batch), 1024, smem, (cudaStream_t)stream>>>(sp);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}
