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
#include <math.h>
#include <new>
#include <stdio.h>
#include <stdlib.h>

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
// PF (prompt prefill): the grid's rows are (token, row) pairs r = tok * rows_real + row at positions P[0] + tok.
// seq_off: length of the condition prefix in front of the tokens; cache position pos reads sequence column pos - seq_off.
template <bool PF>
__global__ void __launch_bounds__(256) lm_embed_kernel(const __half* __restrict__ emb, const float* __restrict__ inv_freq,
                                                       const int64_t* __restrict__ seq, const int* __restrict__ P,
                                                       float* __restrict__ x, int d, int n_q, int card, int max_seq,
                                                       int batch, float pos_scale, int rows_real, bool sin_pos, int seq_off) {
    const int r = blockIdx.x, b = (PF ? r % rows_real : r) % batch, pos = P[0] + (PF ? r / rows_real : 0);
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
            // prefill: row = tk * rows_real + rr -> cache row rr, position cache_pos + tk
            const int which = n >= 2 * p.d ? 2 : (n >= p.d ? 1 : 0), nn = n - which * p.d;
            const int tk = PF ? row / p.rows_real : 0, rr = row - tk * p.rows_real;
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
template <int NPAD>
struct WideCfg {
    static constexpr int W_BYTES = 64 * WIDE_KC * 2;
    static constexpr int STAGE = W_BYTES + NPAD * WIDE_KC * 2;
    static constexpr int STAGES = NPAD <= 128 ? 6 : 5;
    static constexpr int LDS = 68;   // pitch (floats) of the [NPAD][64] fp32 staging tile: conflict-free fragment stores
    static constexpr int SMEM = STAGES * STAGE + 1024 + 64;   // ring (1024-aligned) + barriers
    static_assert(NPAD * LDS * 4 <= STAGES * STAGE, "the staging tile reuses the ring");
};

// EPI is EPI_PARTIAL, EPI_QKV, EPI_QKV_ROPE, EPI_GELU or EPI_F32.  Prefill passes above 64 rows carry one position per row,
// so their QKV epilogue is the decode one (token 0 of the pass at position pos).
template <int NPAD, int EPI>
__global__ void __launch_bounds__(128, 1) lm_gemm_wide_kernel(const __grid_constant__ CUtensorMap wmap,
                                                              const __grid_constant__ CUtensorMap xmap, GemmParams p, int w_row0) {
    using Cfg = WideCfg<NPAD>;
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
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < WIDE_KC / 16; ++kk)   // a 16-element K step advances the start address by 32 bytes
            wgmma_f16<NPAD>(acc, wgmma_desc_sw128(a + 32 * kk), wgmma_desc_sw128(b + 32 * kk), 1u);
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

// ------------------------------------------------------------------------------------------------ attention (1 query)
struct AttnParams {
    const float* q; int q_nsplit; size_t q_split_stride;  // q[s][row][d] fp32 partial sums
    const __half* kc; const __half* vc; __half* out;
    int H, d, cache_len; const int* pos; int fixed_len; float scale;
    int rows_real;                // prefill (PF kernels): rows of the generation
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

// Self attention for one query token: CTA = (query row, head), 8 warps, ONE pass over K and V with an online softmax.  A warp
// instruction covers 4 consecutive cache positions (4 x 128 B = 512 contiguous bytes), 8 lanes share a position (8 dims each).
// Every lane copies its 16-byte slices of K and V with cp.async into a private slot of a per-warp shared-memory ring,
// ATT2_DEPTH iterations deep, and reads them back (its own 32 bytes) one iteration at a time: up to 8 x 32 bytes per lane stay
// outstanding continuously, in shared memory instead of registers.
// PF (prompt prefill): blockIdx.y is a (token, row) pair tok * rows_real + r; the query at position pos + tok attends to the
// cache of row r up to and including its own position (the QKV GEMM of the same pass has already appended every token of the
// pass: causal within the chunk).
constexpr int ATT2_DEPTH = 8;
constexpr int ATT2_SMEM = ATT_WARPS * ATT2_DEPTH * 1024;   // the ring, 64 KB
template <bool PF>
__global__ void __launch_bounds__(ATT_WARPS * 32) lm_attn2_kernel(AttnParams p) {
    extern __shared__ __align__(16) unsigned char att2sm[];   // [warp][depth][K | V][32 lanes][16 B]
    __shared__ float wm[ATT_WARPS], wl[ATT_WARPS], wacc[ATT_WARPS][64];
    const int h = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int qrow = blockIdx.y, row = PF ? qrow % p.rows_real : qrow, tok = PF ? qrow / p.rows_real : 0;
    const int sl = lane & 7, pg = lane >> 3;
    const int n = p.fixed_len > 0 ? p.fixed_len : p.pos[0] + tok + 1;
    const size_t base = ((size_t)row * p.H + h) * p.cache_len * 64 + sl * 8;
    const __half* kb = p.kc + base;
    const __half* vb = p.vc + base;
    const uint32_t ring = smem_u32(att2sm) + (uint32_t)(warp * ATT2_DEPTH * 1024 + lane * 16);
    // iteration k of this warp covers positions (k * 8 + warp) * 4 + pg
    const int n_it = (n + 31 - warp * 4) / 32 > 0 ? (n - warp * 4 + 31) / 32 : 0;   // iterations with at least one live position group
    auto issue = [&](int k) {
        if (k < n_it) {
            const int pp = (k * ATT_WARPS + warp) * 4 + pg;
            if (pp < n) {
                const uint32_t d = ring + (uint32_t)((k % ATT2_DEPTH) * 1024);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(kb + (size_t)pp * 64) : "memory");
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 512u), "l"(vb + (size_t)pp * 64) : "memory");
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
    if (pg == 0) {
        if (sl == 0) { wm[warp] = st.m; wl[warp] = st.l; }
#pragma unroll
        for (int e = 0; e < 8; ++e) wacc[warp][sl * 8 + e] = st.acc[e];
    }
    __syncthreads();
    if (tid < 64) {
        float mx = wm[0];
#pragma unroll
        for (int w = 1; w < ATT_WARPS; ++w) mx = fmaxf(mx, wm[w]);
        float l = 0.f, o = 0.f;
#pragma unroll
        for (int w = 0; w < ATT_WARPS; ++w) {
            const float cw = wm[w] == -INFINITY ? 0.f : __expf(wm[w] - mx);
            l = fmaf(wl[w], cw, l);
            o = fmaf(wacc[w][tid], cw, o);
        }
        p.out[(size_t)qrow * p.d + h * 64 + tid] = __float2half_rn(o / l);
    }
}

// Cross attention over the (short) text condition: one WARP per (row, head), lane = text position for the scores,
// lane = 2 output dims for the weighted sum.  K/V were computed once per generate() (acb_lm_begin).
template <bool PF>
__global__ void __launch_bounds__(256) lm_cross_attn_kernel(AttnParams p, int rows) {
    __shared__ float qs[8][64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pair = blockIdx.x * 8 + warp;          // (row, head) index
    if (pair >= rows * p.H) return;                  // warp-uniform
    const int row = pair / p.H, h = pair % p.H, n = p.fixed_len;
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
    const size_t base = ((size_t)(PF ? row % p.rows_real : row) * p.H + h) * p.cache_len * 64;   // K / V of the generation row
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

__global__ void __launch_bounds__(1024) lm_sample_kernel(SampleParams p) {
    extern __shared__ float sm[];
    float* pr = sm;                 // [card] logits -> probabilities
    float* sv = pr + p.card;        // [NP] sort values
    int* si = (int*)(sv + p.NP);    // [NP] sort indices
    __shared__ float red[3][32];
    __shared__ float bestv[32];
    __shared__ int besti[32];
    __shared__ float s_scalar;
    const int k = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, nt = blockDim.x;
    const int card = p.card;
    const bool cfg = p.rows == 2 * p.batch, cfg3 = p.rows == 3 * p.batch;   // [cond; null] or [cond; style-only; null]
    const float* lc = p.logits + ((size_t)b * p.n_q + k) * card;
    const float* lu = p.logits + ((size_t)((cfg3 ? 2 : 1) * p.batch + b) * p.n_q + k) * card;
    const float* lw = p.logits + ((size_t)(p.batch + b) * p.n_q + k) * card;
    const int cur_pos = p.pos ? p.pos[0] : 0;   // read once: the last block to finish advances it (below)
    const int col = cur_pos - p.seq_off;        // sequence column of the token this step consumed
    const uint32_t step = p.pos ? (uint32_t)col : p.step;

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
                                     : exp1_noise(p.seed, step, (uint32_t)(b * p.n_q + k), (uint32_t)i);
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
    int prefix_len = 0;            // condition-prefix positions in front of the tokens in the KV cache
    const float* prefix = nullptr; // [rows][prefix_len][d] fp32, set only while acb_lm_begin_prefix enqueues the prefix passes
    int launches = 0;
    bool has_cross = false;
    // wide GEMM (max_rows > 64): one map per stacked weight matrix [L * N][K] (encoded by acb_lm_create) and per activation
    // buffer [rows][K] of the current generation (encoded by acb_lm_begin_prefix)
    CUtensorMap wmap[7];
    CUtensorMap xmap_h16, xmap_a16, xmap_f16;
};
enum { WM_QKV = 0, WM_O, WM_CQ, WM_CO, WM_FF1, WM_FF2, WM_HEADS };

static int nt_for_rows(int rows) { return rows <= 8 ? 1 : (rows <= 16 ? 2 : (rows <= 32 ? 4 : 8)); }

static size_t gemm_smem_bytes(int nt, int kslice, int ft2 = 1) {
    return (size_t)16 * ft2 * (kslice * 2 + 64) + 16 + (size_t)4 * 16 * ft2 * (8 * nt + 1) * sizeof(float);
}
constexpr int GEMM_MAX_SMEM = 120 * 1024;

template <int EPI, int FT2>
static int launch_gemm_ft(int nt, const GemmParams& p, int nsplit, cudaStream_t s) {
    dim3 grid(p.N / (16 * FT2), nsplit);
    const size_t smem = gemm_smem_bytes(nt, p.kslice, FT2);
    ACB_REQUIRE(smem <= (size_t)GEMM_MAX_SMEM && p.N % (16 * FT2) == 0, "lm_gemm: tile does not fit (N=%d kslice=%d ft2=%d)", p.N, p.kslice, FT2);
    switch (nt) {
        case 1: lm_gemm_kernel<1, EPI, FT2><<<grid, 128, smem, s>>>(p); break;
        case 2: lm_gemm_kernel<2, EPI, FT2><<<grid, 128, smem, s>>>(p); break;
        case 4: lm_gemm_kernel<4, EPI, FT2><<<grid, 128, smem, s>>>(p); break;
        default: lm_gemm_kernel<8, EPI, FT2><<<grid, 128, smem, s>>>(p); break;
    }
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}
template <int EPI>
static int launch_gemm(int nt, const GemmParams& p, int nsplit, cudaStream_t s, int ft2 = 1) {
    if (ft2 == 2) {
        if constexpr (EPI == EPI_CROSSKV || EPI == EPI_QKV_PF || EPI == EPI_QKV_PF_ROPE) { acb_set_error("lm_gemm: this epilogue uses 16-feature tiles"); return ACB_ERR_INVALID; }
        else return launch_gemm_ft<EPI, 2>(nt, p, nsplit, s);
    }
    return launch_gemm_ft<EPI, 1>(nt, p, nsplit, s);
}

template <int NT, int EPI, int FT2>
static cudaError_t gemm_attr_one() {
    cudaError_t e = cudaFuncSetAttribute(lm_gemm_kernel<NT, EPI, FT2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_MAX_SMEM);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(lm_gemm_kernel<NT, EPI, FT2>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
}
template <int EPI>
static cudaError_t gemm_attr_all() {
    cudaError_t e;
    if ((e = gemm_attr_one<1, EPI, 1>()) != cudaSuccess) return e;
    if ((e = gemm_attr_one<2, EPI, 1>()) != cudaSuccess) return e;
    if ((e = gemm_attr_one<4, EPI, 1>()) != cudaSuccess) return e;
    if ((e = gemm_attr_one<8, EPI, 1>()) != cudaSuccess) return e;
    if constexpr (EPI != EPI_CROSSKV && EPI != EPI_QKV_PF && EPI != EPI_QKV_PF_ROPE) {
        if ((e = gemm_attr_one<1, EPI, 2>()) != cudaSuccess) return e;
        if ((e = gemm_attr_one<2, EPI, 2>()) != cudaSuccess) return e;
        if ((e = gemm_attr_one<4, EPI, 2>()) != cudaSuccess) return e;
        if ((e = gemm_attr_one<8, EPI, 2>()) != cudaSuccess) return e;
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
static int launch_wide(const CUtensorMap& wm, const CUtensorMap& xm, int w_row0, const GemmParams& p, int ny, cudaStream_t s) {
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
    if (wide_npad(p.rows) == 128) {
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
static int enqueue_step(acb_lm* lm, cudaStream_t s, float* logits_out, int* n_launch, bool gemms_only = false,
                        bool capturing = false, int pf_tokens = 0, bool pf_prefix = false) {
    const acb_lm_config& c = lm->cfg;
    const acb_lm_buffers& B = lm->buf;
    const bool pf = pf_tokens > 0;
    ACB_REQUIRE(!pf_prefix || (pf && lm->prefix), "enqueue_step: a prefix pass needs the prefix of acb_lm_begin_prefix");
    const int rows_real = lm->rows, rows = pf ? rows_real * pf_tokens : rows_real;
    const int d = c.dim, ffn = c.ffn_dim, L = c.num_layers, H = c.num_heads, nt = nt_for_rows(rows);
    // rows > 64 (then rows_real > 64 and a prefill pass holds one position per row): every GEMM but EPI_CROSSKV on the wide kernel
    const bool wide = rows > 64;
    const size_t part_stride = (size_t)(pf && !wide ? 8 * nt : lm->rows_pad) * d;
    const size_t kv_layer = (size_t)c.max_rows * H * c.max_seq * 64;
    const size_t ckv_layer = (size_t)c.max_rows * H * c.max_text * 64;
    const float scale = 1.0f / sqrtf(64.f);
    int nl = 0, ks = 0;

    if (!gemms_only) {
        const bool sin_pos = c.positional_embedding != 1;
        if (pf && pf_prefix) lm_embed_prefix_kernel<<<rows, 256, 0, s>>>(lm->prefix, lm->w.inv_freq, B.pos, B.x, d, lm->prefix_len,
                                                                       c.pos_scale, rows_real, sin_pos);
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
    auto partial_gemm = [&](const __half* W, const void* X, int N, int K, int layer, int wm, const CUtensorMap& xm) -> int {
        const int ns = wide ? pick_split_wide(N, K, lm->sms, true, &ks) : pick_split(N, K, lm->sms, true, &ks);
        GemmParams p = base_gemm(W, X, N, K, rows, ks);
        p.out_f32 = B.part; p.ld_out = N; p.split_stride = part_stride;
        if (wide) ACB_TRY(launch_wide<EPI_PARTIAL>(lm->wmap[wm], xm, layer * N, p, ns, s));
        else ACB_TRY(launch_gemm<EPI_PARTIAL>(nt, p, ns, s, pick_ft2(N, K, ns, ks, nt, lm->sms)));
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
            GemmParams p = base_gemm((const __half*)lm->w.w_qkv + (size_t)l * 3 * d * d, B.h16, 3 * d, d, rows, ks);
            p.q32 = B.q32; p.kc = (__half*)B.k_cache + l * kv_layer; p.vc = (__half*)B.v_cache + l * kv_layer;
            p.d = d; p.H = H; p.cache_len = c.max_seq; p.pos = B.pos; p.rows_real = rows_real;
            p.rope_freq = lm->w.rope_freq; p.pos_scale = c.pos_scale;
            const bool rope = c.positional_embedding != 0;
            const int ft2 = pf ? 1 : pick_ft2(3 * d, d, 1, ks, nt, lm->sms);
            if (wide) ACB_TRY(rope ? launch_wide<EPI_QKV_ROPE>(lm->wmap[WM_QKV], lm->xmap_h16, l * 3 * d, p, ns, s)
                                   : launch_wide<EPI_QKV>(lm->wmap[WM_QKV], lm->xmap_h16, l * 3 * d, p, ns, s));
            else if (pf) ACB_TRY(rope ? launch_gemm<EPI_QKV_PF_ROPE>(nt, p, 1, s, ft2) : launch_gemm<EPI_QKV_PF>(nt, p, 1, s, ft2));
            else ACB_TRY(rope ? launch_gemm<EPI_QKV_ROPE>(nt, p, 1, s, ft2) : launch_gemm<EPI_QKV>(nt, p, 1, s, ft2));
            ++nl;
            DBG("gemm_EPI_QKV", l);
        }
        if (!gemms_only) {
            AttnParams a{B.q32, 1, 0, (__half*)B.k_cache + l * kv_layer, (__half*)B.v_cache + l * kv_layer, (__half*)B.a16,
                         H, d, c.max_seq, B.pos, 0, scale, rows_real};
            if (pf) lm_attn2_kernel<true><<<dim3(H, rows), ATT_WARPS * 32, ATT2_SMEM, s>>>(a);
            else lm_attn2_kernel<false><<<dim3(H, rows), ATT_WARPS * 32, ATT2_SMEM, s>>>(a);
            ACB_LAUNCH_CHECK();
            ++nl;
            DBG("lm_attn2_kernel", l);
        }
        ACB_TRY(partial_gemm((const __half*)lm->w.w_o + (size_t)l * d * d, B.a16, d, d, l, WM_O, lm->xmap_a16));
        // --- cross attention
        if (lm->has_cross) {
            ACB_TRY(ln_launch(ln + 2 * d, ln + 3 * d, l));
            ACB_TRY(partial_gemm((const __half*)lm->w.w_cq + (size_t)l * d * d, B.h16, d, d, l, WM_CQ, lm->xmap_h16));
            const int nsq = pending;
            pending = 0;   // these partials are the cross-attention queries, not a residual update
            if (!gemms_only) {
                AttnParams a{B.part, nsq, part_stride, (__half*)B.ck_cache + l * ckv_layer,
                             (__half*)B.cv_cache + l * ckv_layer, (__half*)B.a16, H, d, c.max_text, B.pos, lm->text_len,
                             scale, rows_real};
                if (pf) lm_cross_attn_kernel<true><<<acb_ceil_div(rows * H, 8), 256, 0, s>>>(a, rows);
                else lm_cross_attn_kernel<false><<<acb_ceil_div(rows * H, 8), 256, 0, s>>>(a, rows);
                ACB_LAUNCH_CHECK();
                ++nl;
                DBG("lm_cross_attn_kernel", l);
            }
            ACB_TRY(partial_gemm((const __half*)lm->w.w_co + (size_t)l * d * d, B.a16, d, d, l, WM_CO, lm->xmap_a16));
        }
        // --- feed forward
        ACB_TRY(ln_launch(ln + 4 * d, ln + 5 * d, l));
        {
            const int ns = wide ? pick_split_wide(ffn, d, lm->sms, false, &ks) : pick_split(ffn, d, lm->sms, false, &ks);
            GemmParams p = base_gemm((const __half*)lm->w.w_ff1 + (size_t)l * ffn * d, B.h16, ffn, d, rows, ks);
            p.out_f16 = (__half*)B.f16; p.ld_out = ffn;
            if (wide) ACB_TRY(launch_wide<EPI_GELU>(lm->wmap[WM_FF1], lm->xmap_h16, l * ffn, p, ns, s));
            else ACB_TRY(launch_gemm<EPI_GELU>(nt, p, 1, s, pick_ft2(ffn, d, 1, ks, nt, lm->sms)));
            ++nl;
            DBG("gemm_EPI_GELU", l);
        }
        ACB_TRY(partial_gemm((const __half*)lm->w.w_ff2 + (size_t)l * d * ffn, B.f16, d, ffn, l, WM_FF2, lm->xmap_f16));
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
        lm_sample_kernel<<<dim3(c.n_q, lm->batch), 1024, smem, s>>>(sp);
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
    acb_lm* lm = new (std::nothrow) acb_lm();
    ACB_REQUIRE(lm, "acb_lm_create: out of host memory");
    lm->cfg = *cfg; lm->w = *w; lm->buf = *buf;
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
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT2_SMEM);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT2_SMEM);
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(lm_attn2_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
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
    }
    if (ea != cudaSuccess) {
        acb_set_error("acb_lm_create: cudaFuncSetAttribute: %s", cudaGetErrorString(ea));
        cudaStreamDestroy(lm->capture_stream);
        delete lm;
        return ACB_ERR_CUDA;
    }
    if (cfg->max_rows > 64) {   // the wide GEMM's weight maps: each stacked matrix as [L * N][K], 64-row boxes
        const int d = cfg->dim, ffn = cfg->ffn_dim, L = cfg->num_layers;
        int rc = encode_map(&lm->wmap[WM_QKV], w->w_qkv, d, L * 3 * d, 64);
        if (rc == ACB_OK) rc = encode_map(&lm->wmap[WM_O], w->w_o, d, L * d, 64);
        if (rc == ACB_OK && cfg->cross_attention) rc = encode_map(&lm->wmap[WM_CQ], w->w_cq, d, L * d, 64);
        if (rc == ACB_OK && cfg->cross_attention) rc = encode_map(&lm->wmap[WM_CO], w->w_co, d, L * d, 64);
        if (rc == ACB_OK) rc = encode_map(&lm->wmap[WM_FF1], w->w_ff1, d, L * ffn, 64);
        if (rc == ACB_OK) rc = encode_map(&lm->wmap[WM_FF2], w->w_ff2, ffn, L * d, 64);
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
// the activation buffers zero.
static int prefill_passes(acb_lm* lm, cudaStream_t s, int pos0, int n, bool prefix) {
    const acb_lm_config& c = lm->cfg;
    const int d = c.dim;
    int per = lm->rows > ACB_LM_PREFILL_ROWS ? 1 : ACB_LM_PREFILL_ROWS / lm->rows;
    // ACB_LM_PREFILL_PER=n: at most n positions per pass (n = 1: one position per pass, the reference order for tests)
    if (const char* e = getenv("ACB_LM_PREFILL_PER")) { const int cap = atoi(e); if (cap >= 1 && cap < per) per = cap; }
    int done = 0;
    while (done < n) {
        const int tc = n - done < per ? n - done : per;
        const int vrows = lm->rows * tc, pad = 8 * nt_for_rows(vrows);
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

extern "C" int acb_lm_begin(acb_lm_t* lm, const float* cross, int batch, int rows, int text_len, int seq_len,
                            const acb_lm_sampling* sampling, void* stream) {
    return acb_lm_begin_prefix(lm, cross, nullptr, 0, batch, rows, text_len, seq_len, sampling, stream);
}

extern "C" int acb_lm_begin_prefix(acb_lm_t* lm, const float* cross, const float* prefix, int prefix_len, int batch, int rows,
                                   int text_len, int seq_len, const acb_lm_sampling* sampling, void* stream) {
    ACB_REQUIRE(lm && sampling, "acb_lm_begin: null argument");
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
                GemmParams p = base_gemm((const __half*)lm->w.w_ckv + (size_t)l * 2 * d * d,
                                         (const __half*)lm->buf.cross16 + r0 * d, 2 * d, d, (int)min((size_t)64, M - r0), ks);
                p.kc = (__half*)lm->buf.ck_cache + l * ckv_layer; p.vc = (__half*)lm->buf.cv_cache + l * ckv_layer;
                p.d = d; p.H = H; p.cache_len = c.max_text; p.text_len = text_len; p.row0 = (int)r0;
                ACB_TRY(launch_gemm<EPI_CROSSKV>(8, p, 1, s));
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
    // capture one decode step; its kernels are chained by plain stream-order edges.  (Launched with programmatic dependent launch,
    // the same kernels gave wrong logits on the H100 once the KV cache held more than a few positions, for a cause not found.)
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

// Prompt prefill: consume sequence columns [pos0, pos0 + n_tokens) of every row (their tokens are already in buffers.seq)
// without sampling, ACB_LM_PREFILL_ROWS / rows positions per pass, at cache positions prefix_len + column.  Leaves
// pos = prefix_len + pos0 + n_tokens on the device.
extern "C" int acb_lm_prefill(acb_lm_t* lm, int pos0, int n_tokens, void* stream) {
    ACB_REQUIRE(lm && lm->rows > 0, "acb_lm_prefill: call acb_lm_begin first");
    ACB_REQUIRE(pos0 >= 0 && n_tokens >= 0 && pos0 + n_tokens < lm->seq_len, "acb_lm_prefill: positions [%d, %d) exceed the sequence (%d)",
                pos0, pos0 + n_tokens, lm->seq_len);
    return prefill_passes(lm, (cudaStream_t)stream, lm->prefix_len + pos0, n_tokens, false);
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
