// EnCodec hot path for H100 (sm_90a): SEANet convolutions, LSTM recurrence, residual VQ.
//
// fp32 CUDA-core arithmetic on purpose: RVQ code indices must match the fp32 reference bit for bit on the
// same latent, and a TF32/BF16 tensor-core conv would move the latents by ~1e-3 and flip near-tie codes
// (SURVEY.md section 7 "hard parts").  What is GPU-specific here is the data movement: padding, ELU,
// bias, residual add and the transposed-conv trim are folded into the conv kernels (one read + one write
// of every activation per layer), weight-norm is folded once at load, the [frames x bins] VQ distance
// matrix never leaves the SM, and the LSTM keeps W_hh resident in the 227 KB shared memory of 128 SMs.
#include "common.cuh"
#include "gridbar.cuh"
#include "wgmma.cuh"
#include <stdlib.h>

// ------------------------------------------------------------------------------------------------
// weight-norm fold: w[g][:] = g[g] * v[g][:] / ||v[g]||   (audiocraft/modules/conv.py:21-30)
// ------------------------------------------------------------------------------------------------
__global__ void weight_norm_fold_kernel(const float* __restrict__ v, const float* __restrict__ g,
                                        float* __restrict__ w, int groups, int inner) {
    int grp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (grp >= groups) return;
    const float* vr = v + (size_t)grp * inner;
    float ss = 0.f;
    for (int i = lane; i < inner; i += 32) ss = fmaf(vr[i], vr[i], ss);
    ss = warp_sum(ss);
    float scale = g[grp] / sqrtf(ss);
    for (int i = lane; i < inner; i += 32) w[(size_t)grp * inner + i] = vr[i] * scale;
}

extern "C" int acb_weight_norm_fold(const float* v, const float* g, float* w, int groups, int inner, void* stream) {
    ACB_REQUIRE(v && g && w && groups > 0 && inner > 0, "acb_weight_norm_fold: bad arguments");
    int wpb = 4;
    weight_norm_fold_kernel<<<acb_ceil_div(groups, wpb), wpb * 32, 0, (cudaStream_t)stream>>>(v, g, w, groups, inner);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

// ------------------------------------------------------------------------------------------------
// conv1d: implicit GEMM on fp32 FMA.  CTA tile = (8*CPT output channels) x (32*TPT output steps) of one
// batch item; warp = channel group (weights are warp-broadcast from smem), lane = time (x reads and y
// writes are unit-stride).  The input slab is staged once per input-channel chunk with reflect / zero
// padding and ELU applied on the way in, de-interleaved by stride phase so strided convs read smem
// conflict-free.
// ------------------------------------------------------------------------------------------------
struct ConvParams {
    const float* x; const float* w; const float* bias; const float* res; float* y;
    int c_in, c_out, t_in, t_virt, t_out, K, stride, dil, pad_left, reflect, elu, ci_chunk, span, PL;
    int tr_S, tr_trim, tr_tout;   // transposed conv as a GEMM over virtual channels n' = co*S + phase (conv1d_t5 only)
};

// One warp stages dst[q] = act(x[g0 + q * gstep]) for q in [0, n) (zero beyond, up to n_store): the global loads of 8 lane-strided
// entries are requested before the first is consumed.  A plain `dst[j] = act(load(j))` loop is a chain of dependent L2 round trips
// (the activation branches on the loaded value and the compiler cannot move a load above the shared-memory store before it): that
// pattern was 53 % of conv1d_t6's stall samples and 3x of the fused residual block's run time before it was batched.
__device__ __forceinline__ void stage_span(float* __restrict__ dst, const float* __restrict__ xr, int g0, int gstep, int n, int n_store,
                                           int t_in, int t_virt, int reflect, int elu, int lane) {
    for (int q0 = 0; q0 < n_store; q0 += 256) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int q = q0 + lane + 32 * u;
            int g = g0 + q * gstep;
            if (reflect) {
                if (g < 0) g = -g;
                if (g >= t_virt) g = 2 * (t_virt - 1) - g;
            }
            v[u] = (q < n && g >= 0 && g < t_in) ? __ldg(xr + g) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int q = q0 + lane + 32 * u;
            if (q < n_store) dst[q] = elu ? acb_elu(v[u]) : v[u];
        }
    }
}

template <int CPT, int TPT>
__global__ void __launch_bounds__(256) conv1d_kernel(ConvParams p) {
    constexpr int BM = 8 * CPT, BN = 32 * TPT;
    extern __shared__ float smem[];
    const int XS = p.stride * p.PL;               // floats per staged input channel
    float* ws = smem;                             // [ci_chunk*K][BM]
    float* xs = ws + p.ci_chunk * p.K * BM;       // [ci_chunk][XS]
    int* koff = (int*)(xs + p.ci_chunk * XS);     // [K] tap offset inside a staged channel

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int t0 = blockIdx.x * BN, co0 = blockIdx.y * BM, b = blockIdx.z;
    const float* xb = p.x + (size_t)b * p.c_in * p.t_in;

    if (tid < p.K) {
        int kd = tid * p.dil;
        koff[tid] = (kd % p.stride) * p.PL + kd / p.stride;
    }

    float acc[CPT][TPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i)
#pragma unroll
        for (int j = 0; j < TPT; ++j) acc[i][j] = 0.f;

    const int g0 = t0 * p.stride - p.pad_left;
    for (int ci0 = 0; ci0 < p.c_in; ci0 += p.ci_chunk) {
        const int nci = min(p.ci_chunk, p.c_in - ci0);
        __syncthreads();  // previous chunk fully consumed (also publishes koff on the first pass)
        for (int idx = tid; idx < nci * p.K * BM; idx += 256) {
            int r = idx / BM, c = idx - r * BM;
            ws[idx] = (co0 + c < p.c_out) ? p.w[((size_t)ci0 * p.K + r) * p.c_out + co0 + c] : 0.f;
        }
        // one warp per staged input channel: no integer division in the index math
        for (int cl = warp; cl < nci; cl += 8) {
            const float* xrow = xb + (size_t)(ci0 + cl) * p.t_in;
            float* xdst = xs + cl * XS;
            for (int ph = 0; ph < p.stride; ++ph) {   // stride phase planes (one plane for stride 1)
                const int nq = (p.span - ph + p.stride - 1) / p.stride;
                stage_span(xdst + ph * p.PL, xrow, g0 + ph, p.stride, nq, nq, p.t_in, p.t_virt, p.reflect, p.elu, lane);
            }
        }
        __syncthreads();
        for (int cl = 0; cl < nci; ++cl) {
            const float* xc = xs + cl * XS + lane;
            const float* wc = ws + cl * p.K * BM + warp * CPT;
            for (int k = 0; k < p.K; ++k) {
                float wv[CPT];
#pragma unroll
                for (int i = 0; i < CPT; ++i) wv[i] = wc[k * BM + i];
                const float* xk = xc + koff[k];
#pragma unroll
                for (int j = 0; j < TPT; ++j) {
                    float xv = xk[32 * j];
#pragma unroll
                    for (int i = 0; i < CPT; ++i) acc[i][j] = fmaf(wv[i], xv, acc[i][j]);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < CPT; ++i) {
        int co = co0 + warp * CPT + i;
        if (co >= p.c_out) continue;
        float bv = p.bias ? p.bias[co] : 0.f;
        size_t row = ((size_t)b * p.c_out + co) * p.t_out;
#pragma unroll
        for (int j = 0; j < TPT; ++j) {
            int t = t0 + lane + 32 * j;
            if (t < p.t_out) {
                float v = acc[i][j] + bv;
                if (p.res) v += p.res[row + t];
                p.y[row + t] = v;
            }
        }
    }
}

template <int CPT, int TPT>
static int launch_conv1d(const ConvParams& p, int batch, cudaStream_t s) {
    constexpr int BM = 8 * CPT, BN = 32 * TPT;
    ConvParams q = p;
    q.ci_chunk = max(1, min(p.c_in, 32 / p.K));
    q.span = (BN - 1) * p.stride + (p.K - 1) * p.dil + 1;
    q.PL = acb_ceil_div(q.span, p.stride);
    size_t smem = ((size_t)q.ci_chunk * p.K * BM + (size_t)q.ci_chunk * p.stride * q.PL) * sizeof(float) +
                  p.K * sizeof(int);
    ACB_REQUIRE(smem <= 200 * 1024, "acb_conv1d: tile needs %zu B of shared memory", smem);
    if (smem > 48 * 1024)
        ACB_CHECK_CUDA(cudaFuncSetAttribute(conv1d_kernel<CPT, TPT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem));
    dim3 grid(acb_ceil_div(p.t_out, BN), acb_ceil_div(p.c_out, BM), batch);
    conv1d_kernel<CPT, TPT><<<grid, 256, smem, s>>>(q);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

// ------------------------------------------------------------------------------------------------
// conv1d on the tensor pipe with fp32-level accuracy: 3xTF32.  Every fp32 operand is split into hi = tf32(x) and
// lo = tf32(x - hi); acc += hi*hi + hi*lo + lo*hi (the lo*lo term, 2^-22 relative, is dropped), fp32 accumulate.
// The 3-register FFMA path tops out near 37 TFLOP/s on this part; the tensor pipe does the same implicit GEMM several
// times faster while keeping the latents within ~1e-6 of the fp32 reference (RVQ indices stay put).
// CTA tile 64 output channels x 128 steps, 8 warps as 2 (channels) x 4 (time), warp tile 32 x 32 = 2 x 4 m16n8k8 tiles.
// B fragments are read straight from the staged (padded, ELU'd, phase-de-interleaved) input slab through a per-chunk
// row-offset table, i.e. the im2col matrix is never materialised.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32_(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// fp32 -> tf32, round to nearest, ties away from zero (= cvt.rna.tf32.f32 for every finite input): add half an ulp of the 10-bit
// mantissa to the magnitude bits and clear the 13 dropped bits.  Two integer instructions; the cvt instruction itself is emulated in
// SASS with ~5 (bias add, mask, NaN test + select), and every 3xTF32 operand costs two conversions, so in the mma.sync kernels the
// operand split was ~11 instructions per element against 3 MMAs (lstm_tc_kernel: 96 HMMA among ~900 instructions per 4 k-steps).
// -DACB_CVT_TF32 restores the instruction (NaN payloads are the only difference).
#ifdef ACB_CVT_TF32
__device__ __forceinline__ uint32_t to_tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return r;
}
#else
__device__ __forceinline__ uint32_t to_tf32(float v) { return (__float_as_uint(v) + 0x1000u) & 0xFFFFE000u; }
#endif
// (Handing the low term x - hi to the tensor core unrounded -- it reads only the upper 19 bits of a tf32 operand -- saves two more
//  instructions per element but was measured no faster.  Not kept.)
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

constexpr int TC_BM = 64, TC_BN = 128, TC_WP = TC_BM + 8;   // W smem row pitch = 8 mod 32: conflict-free A fragments

__global__ void __launch_bounds__(256) conv1d_tc_kernel(ConvParams p, int xsp, int rcp) {
    extern __shared__ float smem[];
    float* wh = smem;                          // [rcp][TC_WP] tf32 hi
    float* wl = wh + rcp * TC_WP;              // [rcp][TC_WP] tf32 lo
    float* xs = wl + rcp * TC_WP;              // [ci_chunk][xsp]
    int* roff = (int*)(xs + p.ci_chunk * xsp); // [rcp] slab offset of reduction row r = (channel, tap)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
    const int wm = warp & 1, wn = warp >> 1;
    const int t0 = blockIdx.x * TC_BN, co0 = blockIdx.y * TC_BM, b = blockIdx.z;
    const float* xb = p.x + (size_t)b * p.c_in * p.t_in;

    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;

    const int g0 = t0 * p.stride - p.pad_left;
    for (int ci0 = 0; ci0 < p.c_in; ci0 += p.ci_chunk) {
        const int nci = min(p.ci_chunk, p.c_in - ci0);
        const int rc = nci * p.K, rcu = (rc + 7) & ~7;
        __syncthreads();
        for (int idx = tid; idx < rcu * TC_BM; idx += 256) {
            const int r = idx / TC_BM, cc = idx - r * TC_BM;
            const float w = (r < rc && co0 + cc < p.c_out) ? p.w[((size_t)ci0 * p.K + r) * p.c_out + co0 + cc] : 0.f;
            const uint32_t hi = to_tf32(w);
            wh[r * TC_WP + cc] = __uint_as_float(hi);
            wl[r * TC_WP + cc] = __uint_as_float(to_tf32(w - __uint_as_float(hi)));
        }
        for (int r = tid; r < rcu; r += 256) {
            int off = 0;
            if (r < rc) {
                const int cl = r / p.K, k = r - cl * p.K, kd = k * p.dil;
                off = cl * xsp + (kd % p.stride) * p.PL + kd / p.stride;
            }
            roff[r] = off;
        }
        for (int cl = warp; cl < nci; cl += 8) {
            const float* xrow = xb + (size_t)(ci0 + cl) * p.t_in;
            float* xdst = xs + cl * xsp;
            for (int ph = 0; ph < p.stride; ++ph) {
                const int nq = (p.span - ph + p.stride - 1) / p.stride;
                stage_span(xdst + ph * p.PL, xrow, g0 + ph, p.stride, nq, nq, p.t_in, p.t_virt, p.reflect, p.elu, lane);
            }
        }
        __syncthreads();
        const float* xw = xs + wn * 32 + g;
        for (int kk = 0; kk < rcu; kk += 8) {
            uint32_t ah[2][4], al[2][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const int m = wm * 32 + mt * 16 + g;
                ah[mt][0] = __float_as_uint(wh[(kk + c) * TC_WP + m]);
                ah[mt][1] = __float_as_uint(wh[(kk + c) * TC_WP + m + 8]);
                ah[mt][2] = __float_as_uint(wh[(kk + c + 4) * TC_WP + m]);
                ah[mt][3] = __float_as_uint(wh[(kk + c + 4) * TC_WP + m + 8]);
                al[mt][0] = __float_as_uint(wl[(kk + c) * TC_WP + m]);
                al[mt][1] = __float_as_uint(wl[(kk + c) * TC_WP + m + 8]);
                al[mt][2] = __float_as_uint(wl[(kk + c + 4) * TC_WP + m]);
                al[mt][3] = __float_as_uint(wl[(kk + c + 4) * TC_WP + m + 8]);
            }
            const int o0 = roff[kk + c], o1 = roff[kk + c + 4];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const float x0 = xw[o0 + nt * 8], x1 = xw[o1 + nt * 8];
                const uint32_t bh0 = to_tf32(x0), bh1 = to_tf32(x1);
                const uint32_t bl0 = to_tf32(x0 - __uint_as_float(bh0)), bl1 = to_tf32(x1 - __uint_as_float(bh1));
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    mma_tf32(acc[mt][nt], al[mt], bh0, bh1);
                    mma_tf32(acc[mt][nt], ah[mt], bl0, bl1);
                    mma_tf32(acc[mt][nt], ah[mt], bh0, bh1);
                }
            }
        }
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int co = co0 + wm * 32 + mt * 16 + g + 8 * hrow;
            if (co >= p.c_out) continue;
            const float bv = p.bias ? p.bias[co] : 0.f;
            const size_t row = ((size_t)b * p.c_out + co) * p.t_out;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int t = t0 + wn * 32 + nt * 8 + 2 * c + e;
                    if (t < p.t_out) {
                        float v = acc[mt][nt][2 * hrow + e] + bv;
                        if (p.res) v += p.res[row + t];
                        p.y[row + t] = v;
                    }
                }
        }
}

static int launch_conv1d_tc(const ConvParams& p, int batch, cudaStream_t s) {
    ConvParams q = p;
    q.ci_chunk = max(1, min(p.c_in, 32 / p.K));
    q.span = (TC_BN - 1) * p.stride + (p.K - 1) * p.dil + 1;
    q.PL = acb_ceil_div(q.span, p.stride);
    int xsp = p.stride * q.PL;
    xsp += (8 - (xsp & 31) + 32) & 31;            // channel pitch = 8 mod 32: conflict-free B fragments
    const int rcp = (q.ci_chunk * p.K + 7) & ~7;
    size_t smem = ((size_t)2 * rcp * TC_WP + (size_t)q.ci_chunk * xsp) * sizeof(float) + rcp * sizeof(int);
    ACB_REQUIRE(smem <= 200 * 1024, "acb_conv1d: tensor-core tile needs %zu B of shared memory", smem);
    if (smem > 48 * 1024)
        ACB_CHECK_CUDA(cudaFuncSetAttribute(conv1d_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(acb_ceil_div(p.t_out, TC_BN), acb_ceil_div(p.c_out, TC_BM), batch);
    conv1d_tc_kernel<<<grid, 256, smem, s>>>(q, xsp, rcp);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

// ------------------------------------------------------------------------------------------------
// SEANetResnetBlock with the identity skip (audiocraft/modules/seanet.py:44-69, true_skip=True) as ONE kernel:
//     y = x + W2 . elu(b1 + W1 * elu(x)) + b2          W1: k=3 conv C -> C/2,  W2: 1x1 conv C/2 -> C
// As two layer kernels the block moves x, the hidden tensor (twice) and y through HBM (4 C-equivalents + 1.5 C of hidden traffic)
// and is bandwidth / latency bound at 64-128 channels.  Here a CTA owns 128 time steps
// of one item: the ELU'd input slab [C][128 + 2 dil] is staged once, GEMM 1 (M = C/2 hidden channels, N = 128 steps, K = 3C; W1
// streamed in chunks of 16 input channels x 3 taps) leaves the hidden tile in registers, bias + ELU moves it to shared memory (over
// the slab), GEMM 2 (M = C in chunks of 64 output channels, K = C/2) reads it from there and the epilogue adds bias and the skip.
// HBM traffic: x once (+ a second L2-hot read for the skip), y once.  Arithmetic: 3xTF32 on mma.sync.m16n8k8 (hi*lo + lo*hi + hi*hi).
// FLUSH (encoder: RVQ indices must not move): tensor-core accumulation runs over 8 input channels x 3 taps (resp. 16 hidden
// channels) only and is then added to fp32 registers, as in conv1d_t6 -- the tensor core's own accumulate rounding is what costs
// index parity on long reductions, not the operand split.
// Reduction rows of GEMM 1 are ordered (tap, channel): the 8 rows of one k-step are 8 channels at one tap, so with the slab pitch
// = 8 mod 32 the B-fragment reads are bank-conflict free.
// ------------------------------------------------------------------------------------------------
constexpr int RB_TB = 128, RB_XSP = 136, RB_CH = 16;
struct ResblockParams {
    const float* x; const float* w1; const float* b1; const float* w2; const float* b2; float* y;
    int T, dil, pad_left, reflect;
};

__device__ __forceinline__ void rb_split(float v, uint32_t& hi, uint32_t& lo) {
    hi = to_tf32(v);
    lo = to_tf32(v - __uint_as_float(hi));
}

template <int HD, bool FLUSH>
__global__ void __launch_bounds__(HD >= 128 ? 512 : 256, HD >= 128 ? 1 : 2) resblock_kernel(ResblockParams p) {
    // 256 threads (8 warps) up to 128 channels, 512 (16 warps) at 256 channels: GEMM 1 tiles the hidden channels over WM1 warp rows
    // of MT1 m16 tiles and 4 warp columns of 32 steps; GEMM 2 (64 output channels per pass) uses 2 warp rows x WN2 warp columns.
    constexpr int NTHR = HD >= 128 ? 512 : 256, NWARP = NTHR / 32, WM1 = NWARP / 4, MT1 = HD / (16 * WM1), WN2 = NWARP / 2, NT2 = 16 / WN2;
    constexpr int C = 2 * HD, WP1 = HD + 8, WP2 = 64 + 8;
    constexpr bool EARLY_SKIP = !FLUSH || HD == 32;   // skip-connection loads before the MMAs of a pass (registers permitting) or after
    constexpr bool PF_W2 = !(FLUSH && HD == 64);      // next W2 chunk prefetched into registers during the MMAs (registers permitting)
    constexpr int WHALF = (3 * RB_CH * WP1) > (HD * WP2) ? (3 * RB_CH * WP1) : (HD * WP2);
    constexpr int NSL = C * RB_XSP / NTHR, SLB = 34;   // slab elements per thread (34 / 68 / 68), requested 34 at a time (ncu: 21 % of the
                                                       // stall samples were the first use of a 17-element batch, twice per tile at 64 channels)
    constexpr int NW1 = 3 * RB_CH * HD / NTHR;         // W1 chunk elements per thread (6 / 12 / 24)
    constexpr int NW2 = HD * 64 / NTHR;                // W2 chunk elements per thread (8 / 16 / 32)
    static_assert(NSL % SLB == 0 && C * RB_XSP % NTHR == 0, "slab staging");
    extern __shared__ float rsm[];
    float* xs = rsm;                 // [C][RB_XSP] elu(x); after GEMM 1: [HD][RB_XSP] elu(hidden)
    float* wh = xs + C * RB_XSP;     // weight chunk, tf32 hi
    float* wl = wh + WHALF;          // weight chunk, tf32 lo

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
    const int wm = warp % WM1, wn = warp / WM1;     // GEMM 1
    const int wm2 = warp & 1, wn2 = warp >> 1;      // GEMM 2
    const int t0 = blockIdx.x * RB_TB, b = blockIdx.y;
    const float* __restrict__ xb = p.x + (size_t)b * C * p.T;
    const float* __restrict__ w1g = p.w1;
    const float* __restrict__ w2g = p.w2;
    const int span = RB_TB + 2 * p.dil;

    // Every global read below is requested in batches BEFORE anything of the batch is consumed or stored: a load -> store -> load
    // chain through shared memory (the compiler has to assume aliasing) costs one L2 round trip per element.
    float w1r[NW1];
    auto load_w1 = [&](int ci0) {
#pragma unroll
        for (int i = 0; i < NW1; ++i) {
            const int idx = tid + NTHR * i, r = idx / HD, m = idx - r * HD, tap = r / RB_CH, cl = r - tap * RB_CH;
            w1r[i] = __ldg(w1g + ((size_t)tap * C + ci0 + cl) * HD + m);
        }
    };
    load_w1(0);
#pragma unroll 1
    for (int i0 = 0; i0 < NSL; i0 += SLB) {
        float v[SLB];
#pragma unroll
        for (int i = 0; i < SLB; ++i) {
            const int idx = tid + NTHR * (i0 + i), ch = idx / RB_XSP, j = idx - ch * RB_XSP;
            int gt = t0 - p.pad_left + j;
            if (p.reflect) {
                if (gt < 0) gt = -gt;
                if (gt >= p.T) gt = 2 * (p.T - 1) - gt;
            }
            v[i] = (j < span && gt >= 0 && gt < p.T) ? __ldg(xb + (size_t)ch * p.T + gt) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < SLB; ++i) xs[tid + NTHR * (i0 + i)] = acb_elu(v[i]);
    }

    float acc1[MT1][4][4];
#pragma unroll
    for (int i = 0; i < MT1; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc1[i][j][0] = acc1[i][j][1] = acc1[i][j][2] = acc1[i][j][3] = 0.f;

#pragma unroll 1
    for (int ci0 = 0; ci0 < C; ci0 += RB_CH) {
        __syncthreads();   // slab complete (first pass) / previous weight chunk consumed
#pragma unroll
        for (int i = 0; i < NW1; ++i) {
            const int idx = tid + NTHR * i, r = idx / HD, m = idx - r * HD;
            uint32_t hi, lo;
            rb_split(w1r[i], hi, lo);
            wh[r * WP1 + m] = __uint_as_float(hi);
            wl[r * WP1 + m] = __uint_as_float(lo);
        }
        __syncthreads();
        if (ci0 + RB_CH < C) load_w1(ci0 + RB_CH);   // next chunk's weights fly during this chunk's MMAs
#pragma unroll
        for (int c8 = 0; c8 < RB_CH / 8; ++c8) {
            float accc[MT1][4][4];
            if (FLUSH) {
#pragma unroll
                for (int i = 0; i < MT1; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) accc[i][j][0] = accc[i][j][1] = accc[i][j][2] = accc[i][j][3] = 0.f;
            }
#pragma unroll
            for (int tap = 0; tap < 3; ++tap) {
                const int kr = tap * RB_CH + c8 * 8;
                uint32_t ah[MT1][4], al[MT1][4];
#pragma unroll
                for (int mt = 0; mt < MT1; ++mt) {
                    const int m = wm * (16 * MT1) + mt * 16 + g;
                    ah[mt][0] = __float_as_uint(wh[(kr + c) * WP1 + m]);
                    ah[mt][1] = __float_as_uint(wh[(kr + c) * WP1 + m + 8]);
                    ah[mt][2] = __float_as_uint(wh[(kr + c + 4) * WP1 + m]);
                    ah[mt][3] = __float_as_uint(wh[(kr + c + 4) * WP1 + m + 8]);
                    al[mt][0] = __float_as_uint(wl[(kr + c) * WP1 + m]);
                    al[mt][1] = __float_as_uint(wl[(kr + c) * WP1 + m + 8]);
                    al[mt][2] = __float_as_uint(wl[(kr + c + 4) * WP1 + m]);
                    al[mt][3] = __float_as_uint(wl[(kr + c + 4) * WP1 + m + 8]);
                }
                const float* x0p = xs + (ci0 + c8 * 8 + c) * RB_XSP + tap * p.dil + wn * 32 + g;
                const float* x1p = x0p + 4 * RB_XSP;
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    uint32_t bh0, bl0, bh1, bl1;
                    rb_split(x0p[nt * 8], bh0, bl0);
                    rb_split(x1p[nt * 8], bh1, bl1);
#pragma unroll
                    for (int mt = 0; mt < MT1; ++mt) {
                        float (&d)[4] = FLUSH ? accc[mt][nt] : acc1[mt][nt];
                        mma_tf32(d, al[mt], bh0, bh1);
                        mma_tf32(d, ah[mt], bl0, bl1);
                        mma_tf32(d, ah[mt], bh0, bh1);
                    }
                }
            }
            if (FLUSH) {
#pragma unroll
                for (int i = 0; i < MT1; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        acc1[i][j][0] += accc[i][j][0]; acc1[i][j][1] += accc[i][j][1];
                        acc1[i][j][2] += accc[i][j][2]; acc1[i][j][3] += accc[i][j][3];
                    }
            }
        }
    }
    float w2r[NW2];
    auto load_w2 = [&](int co0) {
#pragma unroll
        for (int i = 0; i < NW2; ++i) {
            const int idx = tid + NTHR * i, r = idx >> 6, m = idx & 63;
            w2r[i] = __ldg(w2g + (size_t)r * C + co0 + m);
        }
    };
    if (PF_W2) load_w2(0);
    __syncthreads();   // every warp is done with the slab and the last W1 chunk
    // hidden tile -> shared memory (bias + ELU), over the slab
#pragma unroll
    for (int mt = 0; mt < MT1; ++mt)
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int m = wm * (16 * MT1) + mt * 16 + g + 8 * hrow;
            const float bv = __ldg(p.b1 + m);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int t = wn * 32 + nt * 8 + 2 * c;
                *reinterpret_cast<float2*>(xs + m * RB_XSP + t) =
                    make_float2(acb_elu(acc1[mt][nt][2 * hrow] + bv), acb_elu(acc1[mt][nt][2 * hrow + 1] + bv));
            }
        }

    const bool pair_ok = (p.T & 1) == 0;   // row bases even -> the (t, t+1) pairs of the epilogue are 8-byte aligned
#pragma unroll 1
    for (int co0 = 0; co0 < C; co0 += 64) {
        if (co0) __syncthreads();   // previous W2 chunk consumed
        if (!PF_W2) load_w2(co0);
#pragma unroll
        for (int i = 0; i < NW2; ++i) {
            const int idx = tid + NTHR * i, r = idx >> 6, m = idx & 63;
            uint32_t hi, lo;
            rb_split(w2r[i], hi, lo);
            wh[r * WP2 + m] = __uint_as_float(hi);
            wl[r * WP2 + m] = __uint_as_float(lo);
        }
        __syncthreads();   // W2 chunk (and, first pass, the hidden tile) visible
        if (PF_W2 && co0 + 64 < C) load_w2(co0 + 64);
        // the skip connection under this warp's output tile
        float2 xsk[2][2][NT2];
        auto load_skip = [&]() {
    #pragma unroll
            for (int mt = 0; mt < 2; ++mt)
    #pragma unroll
                for (int hrow = 0; hrow < 2; ++hrow) {
                    const int co = co0 + wm2 * 32 + mt * 16 + g + 8 * hrow;
                    const float* __restrict__ xr = xb + (size_t)co * p.T;
    #pragma unroll
                    for (int nt = 0; nt < NT2; ++nt) {
                        const int t = t0 + wn2 * (8 * NT2) + nt * 8 + 2 * c;
                        if (pair_ok && t + 1 < p.T) xsk[mt][hrow][nt] = __ldg(reinterpret_cast<const float2*>(xr + t));
                        else xsk[mt][hrow][nt] = make_float2(t < p.T ? __ldg(xr + t) : 0.f, t + 1 < p.T ? __ldg(xr + t + 1) : 0.f);
                    }
                }
        };
        if (EARLY_SKIP) load_skip();
        float acc2[2][NT2][4];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < NT2; ++j) acc2[i][j][0] = acc2[i][j][1] = acc2[i][j][2] = acc2[i][j][3] = 0.f;
#pragma unroll 1
        for (int kk = 0; kk < HD; kk += 16) {
            float accc[2][NT2][4];
            if (FLUSH) {
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int j = 0; j < NT2; ++j) accc[i][j][0] = accc[i][j][1] = accc[i][j][2] = accc[i][j][3] = 0.f;
            }
#pragma unroll
            for (int k8 = 0; k8 < 16; k8 += 8) {
                const int kr = kk + k8;
                uint32_t ah[2][4], al[2][4];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    const int m = wm2 * 32 + mt * 16 + g;
                    ah[mt][0] = __float_as_uint(wh[(kr + c) * WP2 + m]);
                    ah[mt][1] = __float_as_uint(wh[(kr + c) * WP2 + m + 8]);
                    ah[mt][2] = __float_as_uint(wh[(kr + c + 4) * WP2 + m]);
                    ah[mt][3] = __float_as_uint(wh[(kr + c + 4) * WP2 + m + 8]);
                    al[mt][0] = __float_as_uint(wl[(kr + c) * WP2 + m]);
                    al[mt][1] = __float_as_uint(wl[(kr + c) * WP2 + m + 8]);
                    al[mt][2] = __float_as_uint(wl[(kr + c + 4) * WP2 + m]);
                    al[mt][3] = __float_as_uint(wl[(kr + c + 4) * WP2 + m + 8]);
                }
                const float* h0p = xs + (kr + c) * RB_XSP + wn2 * (8 * NT2) + g;
                const float* h1p = h0p + 4 * RB_XSP;
#pragma unroll
                for (int nt = 0; nt < NT2; ++nt) {
                    uint32_t bh0, bl0, bh1, bl1;
                    rb_split(h0p[nt * 8], bh0, bl0);
                    rb_split(h1p[nt * 8], bh1, bl1);
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) {
                        float (&d)[4] = FLUSH ? accc[mt][nt] : acc2[mt][nt];
                        mma_tf32(d, al[mt], bh0, bh1);
                        mma_tf32(d, ah[mt], bl0, bl1);
                        mma_tf32(d, ah[mt], bh0, bh1);
                    }
                }
            }
            if (FLUSH) {
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int j = 0; j < NT2; ++j) {
                        acc2[i][j][0] += accc[i][j][0]; acc2[i][j][1] += accc[i][j][1];
                        acc2[i][j][2] += accc[i][j][2]; acc2[i][j][3] += accc[i][j][3];
                    }
            }
        }
        if (!EARLY_SKIP) load_skip();
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int hrow = 0; hrow < 2; ++hrow) {
                const int co = co0 + wm2 * 32 + mt * 16 + g + 8 * hrow;
                const float bv = __ldg(p.b2 + co);
                float* yr = p.y + ((size_t)b * C + co) * p.T;
#pragma unroll
                for (int nt = 0; nt < NT2; ++nt) {
                    const int t = t0 + wn2 * (8 * NT2) + nt * 8 + 2 * c;
                    const float v0 = acc2[mt][nt][2 * hrow] + bv + xsk[mt][hrow][nt].x;
                    const float v1 = acc2[mt][nt][2 * hrow + 1] + bv + xsk[mt][hrow][nt].y;
                    if (pair_ok && t + 1 < p.T) {
                        *reinterpret_cast<float2*>(yr + t) = make_float2(v0, v1);
                    } else {
                        if (t < p.T) yr[t] = v0;
                        if (t + 1 < p.T) yr[t + 1] = v1;
                    }
                }
            }
    }
}

// ------------------------------------------------------------------------------------------------
// resblock_kernel with both GEMM operands split into two fp16 terms instead of two tf32 terms (x = hi + lo 2^-11, hi = fp16(x),
// lo = fp16((x - hi) 2^11): 22 mantissa bits, the class of the tf32 split; activations and folded weights of the codec sit well inside
// fp16's range).  A 16-element reduction step is 3 mma.sync.m16n8k16 (hi.hi | hi.lo + lo.hi into a second accumulator that is scaled
// by 2^-11 when it is folded in) instead of 6 m16n8k8, and the split happens ONCE per element while staging -- weights into half2
// pairs of consecutive reduction rows [k pair][m], the ELU'd slab and the hidden tile into half2 pairs of consecutive channels
// [channel pair][step] -- so the inner loops are LDS + HMMA only (the tf32 kernel: ~10 split instructions per B element and use).
// Same tiling, chunking, epilogue and FLUSH rule (a tensor-core accumulation run covers 16 input channels x 3 taps, resp. 16 hidden
// channels, then goes to fp32 registers) as resblock_kernel.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_f16r(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// two values -> (half2 of the high terms, half2 of the scaled low terms); .x = first value (even reduction index)
__device__ __forceinline__ void split2_h2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(v0, v1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn((v0 - hf.x) * 2048.f, (v1 - hf.y) * 2048.f);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

template <int HD, bool FLUSH>
__global__ void __launch_bounds__(HD >= 128 ? 512 : 256, HD >= 128 ? 1 : 2) resblock_h2_kernel(ResblockParams p) {
    constexpr int NTHR = HD >= 128 ? 512 : 256, NWARP = NTHR / 32, WM1 = NWARP / 4, MT1 = HD / (16 * WM1), WN2 = NWARP / 2, NT2 = 16 / WN2;
    constexpr int C = 2 * HD, WP1 = HD + 8, WP2 = 64 + 8;
    constexpr int KP1 = 3 * RB_CH / 2;                 // k pairs of a W1 chunk (16 channels x 3 taps)
    constexpr int WHALF = (KP1 * WP1) > ((HD / 2) * WP2) ? (KP1 * WP1) : ((HD / 2) * WP2);
    constexpr int NPR = (C / 2) * RB_XSP / NTHR, SLB = 17;   // slab channel PAIRS per thread (17 / 34 / 34), 17 pairs = 34 loads at a time
    constexpr int NW1 = KP1 * HD / NTHR;               // W1 chunk k pairs per thread (3 / 6 / 6)
    constexpr int NW2 = (HD / 2) * 64 / NTHR;          // W2 chunk k pairs per thread (4 / 8 / 8)
    constexpr float LO = 1.f / 2048.f;
    static_assert(NPR % SLB == 0 && (C / 2) * RB_XSP % NTHR == 0 && KP1 * HD % NTHR == 0, "staging");
    extern __shared__ uint32_t rsm2[];
    uint32_t* xh = rsm2;                       // [C/2][RB_XSP] half2 (channel 2i, 2i+1) high terms; after GEMM 1: hidden tile [HD/2][RB_XSP]
    uint32_t* xl = xh + (C / 2) * RB_XSP;      // ... low terms (x 2^11)
    uint32_t* wh = xl + (C / 2) * RB_XSP;      // weight chunk [k pair][m], high terms
    uint32_t* wl = wh + WHALF;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
    const int wm = warp % WM1, wn = warp / WM1;     // GEMM 1
    const int wm2 = warp & 1, wn2 = warp >> 1;      // GEMM 2
    const int t0 = blockIdx.x * RB_TB, b = blockIdx.y;
    const float* __restrict__ xb = p.x + (size_t)b * C * p.T;
    const float* __restrict__ w1g = p.w1;
    const float* __restrict__ w2g = p.w2;
    const int span = RB_TB + 2 * p.dil;

    float w1r[NW1][2];
    auto load_w1 = [&](int ci0) {   // chunk row (tap, cl): k pair (tap, cl / 2) = channels ci0 + 2 j, 2 j + 1 at one tap
#pragma unroll
        for (int i = 0; i < NW1; ++i) {
            const int idx = tid + NTHR * i, kp = idx / HD, m = idx - kp * HD, tap = kp / (RB_CH / 2), j = kp - tap * (RB_CH / 2);
            const float* src = w1g + ((size_t)tap * C + ci0 + 2 * j) * HD + m;
            w1r[i][0] = __ldg(src);
            w1r[i][1] = __ldg(src + HD);
        }
    };
    load_w1(0);
#pragma unroll 1
    for (int i0 = 0; i0 < NPR; i0 += SLB) {
        float v[SLB][2];
#pragma unroll
        for (int i = 0; i < SLB; ++i) {
            const int idx = tid + NTHR * (i0 + i), cp = idx / RB_XSP, j = idx - cp * RB_XSP;
            int gt = t0 - p.pad_left + j;
            if (p.reflect) {
                if (gt < 0) gt = -gt;
                if (gt >= p.T) gt = 2 * (p.T - 1) - gt;
            }
            const bool ok = j < span && gt >= 0 && gt < p.T;
            v[i][0] = ok ? __ldg(xb + (size_t)(2 * cp) * p.T + gt) : 0.f;
            v[i][1] = ok ? __ldg(xb + (size_t)(2 * cp + 1) * p.T + gt) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < SLB; ++i) {
            uint32_t hi, lo;
            split2_h2(acb_elu(v[i][0]), acb_elu(v[i][1]), hi, lo);
            xh[tid + NTHR * (i0 + i)] = hi;
            xl[tid + NTHR * (i0 + i)] = lo;
        }
    }

    float acc1[MT1][4][4];                     // FLUSH: fp32 totals; else: the hi.hi accumulators
    float accx[FLUSH ? 1 : MT1][4][4];         // !FLUSH: the cross-term accumulators (x 2^11)
#pragma unroll
    for (int i = 0; i < MT1; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc1[i][j][0] = acc1[i][j][1] = acc1[i][j][2] = acc1[i][j][3] = 0.f;
    if (!FLUSH) {
#pragma unroll
        for (int i = 0; i < MT1; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) accx[i][j][0] = accx[i][j][1] = accx[i][j][2] = accx[i][j][3] = 0.f;
    }

#pragma unroll 1
    for (int ci0 = 0; ci0 < C; ci0 += RB_CH) {
        __syncthreads();   // slab complete (first pass) / previous weight chunk consumed
#pragma unroll
        for (int i = 0; i < NW1; ++i) {
            const int idx = tid + NTHR * i, kp = idx / HD, m = idx - kp * HD;
            uint32_t hi, lo;
            split2_h2(w1r[i][0], w1r[i][1], hi, lo);
            wh[kp * WP1 + m] = hi;
            wl[kp * WP1 + m] = lo;
        }
        __syncthreads();
        if (ci0 + RB_CH < C) load_w1(ci0 + RB_CH);   // next chunk's weights fly during this chunk's MMAs
        // FLUSH: a run (this chunk: 3 taps x 16 channels) accumulates in c0 (hi.hi) / c1 (cross terms x 2^11) for one m tile and TWO of
        // the warp's four n tiles at a time (16 registers; with all four live the 64- / 128-hidden-channel variants spilled), then folds
        // into the fp32 totals.  Not FLUSH: straight into acc1 / accx, all four n tiles per A fragment.
        constexpr int NH = FLUSH ? 2 : 1, NTH = 4 / NH;
#pragma unroll
        for (int mt = 0; mt < MT1; ++mt) {
            const int m = wm * (16 * MT1) + mt * 16 + g;
#pragma unroll
            for (int nh = 0; nh < NH; ++nh) {
                float c0[NTH][4], c1[NTH][4];
                if (FLUSH) {
#pragma unroll
                    for (int j = 0; j < NTH; ++j) {
                        c0[j][0] = c0[j][1] = c0[j][2] = c0[j][3] = 0.f;
                        c1[j][0] = c1[j][1] = c1[j][2] = c1[j][3] = 0.f;
                    }
                }
#pragma unroll
                for (int tap = 0; tap < 3; ++tap) {
                    const int kr = tap * (RB_CH / 2);
                    uint32_t ah[4], al[4];           // a0 = (m, k pair c), a1 = (m + 8, c), a2 = (m, c + 4), a3 = (m + 8, c + 4)
                    ah[0] = wh[(kr + c) * WP1 + m];     ah[1] = wh[(kr + c) * WP1 + m + 8];
                    ah[2] = wh[(kr + c + 4) * WP1 + m]; ah[3] = wh[(kr + c + 4) * WP1 + m + 8];
                    al[0] = wl[(kr + c) * WP1 + m];     al[1] = wl[(kr + c) * WP1 + m + 8];
                    al[2] = wl[(kr + c + 4) * WP1 + m]; al[3] = wl[(kr + c + 4) * WP1 + m + 8];
                    const int xo = (ci0 / 2 + c) * RB_XSP + tap * p.dil + wn * 32 + g;   // b0 = (k pair c, step g), b1 = (k pair c + 4, g)
#pragma unroll
                    for (int j = 0; j < NTH; ++j) {
                        const int nt = nh * NTH + j;
                        const uint32_t bh0 = xh[xo + nt * 8], bh1 = xh[xo + 4 * RB_XSP + nt * 8];
                        const uint32_t bl0 = xl[xo + nt * 8], bl1 = xl[xo + 4 * RB_XSP + nt * 8];
                        float (&d0)[4] = FLUSH ? c0[j] : acc1[mt][nt];
                        float (&d1)[4] = FLUSH ? c1[j] : accx[FLUSH ? 0 : mt][nt];
                        mma_f16r(d0, ah, bh0, bh1);
                        mma_f16r(d1, ah, bl0, bl1);
                        mma_f16r(d1, al, bh0, bh1);
                    }
                }
                if (FLUSH) {
#pragma unroll
                    for (int j = 0; j < NTH; ++j)
#pragma unroll
                        for (int e = 0; e < 4; ++e) acc1[mt][nh * NTH + j][e] += fmaf(c1[j][e], LO, c0[j][e]);
                }
            }
        }
    }
    if (!FLUSH) {
#pragma unroll
        for (int i = 0; i < MT1; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc1[i][j][e] = fmaf(accx[i][j][e], LO, acc1[i][j][e]);
    }
    float w2r[NW2][2];
    auto load_w2 = [&](int co0) {
#pragma unroll
        for (int i = 0; i < NW2; ++i) {
            const int idx = tid + NTHR * i, kp = idx >> 6, m = idx & 63;
            const float* src = w2g + (size_t)(2 * kp) * C + co0 + m;
            w2r[i][0] = __ldg(src);
            w2r[i][1] = __ldg(src + C);
        }
    };
    load_w2(0);
    __syncthreads();   // every warp is done with the slab and the last W1 chunk
    // hidden tile -> shared memory (bias + ELU + split), over the slab, as half2 pairs of consecutive hidden channels: rows m (lane
    // group g) and m + 1 (g + 1) sit 4 lanes apart; the even row's lane packs step 2c, the odd row's lane step 2c + 1.
#pragma unroll
    for (int mt = 0; mt < MT1; ++mt)
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int m = wm * (16 * MT1) + mt * 16 + g + 8 * hrow;
            const float bv = __ldg(p.b1 + m);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const float v0 = acb_elu(acc1[mt][nt][2 * hrow] + bv), v1 = acb_elu(acc1[mt][nt][2 * hrow + 1] + bv);
                const bool even = (g & 1) == 0;
                const float recv = __shfl_xor_sync(0xffffffffu, even ? v1 : v0, 4);   // partner row's value at the step this lane packs
                uint32_t hi, lo;
                if (even) split2_h2(v0, recv, hi, lo);     // (row m, row m + 1) at step 2c
                else split2_h2(recv, v1, hi, lo);          // (row m - 1, row m) at step 2c + 1
                const int t = wn * 32 + nt * 8 + 2 * c + (even ? 0 : 1);
                xh[(m >> 1) * RB_XSP + t] = hi;
                xl[(m >> 1) * RB_XSP + t] = lo;
            }
        }

    const bool pair_ok = (p.T & 1) == 0;   // row bases even -> the (t, t+1) pairs of the epilogue are 8-byte aligned
#pragma unroll 1
    for (int co0 = 0; co0 < C; co0 += 64) {
        if (co0) __syncthreads();   // previous W2 chunk consumed
#pragma unroll
        for (int i = 0; i < NW2; ++i) {
            const int idx = tid + NTHR * i, kp = idx >> 6, m = idx & 63;
            uint32_t hi, lo;
            split2_h2(w2r[i][0], w2r[i][1], hi, lo);
            wh[kp * WP2 + m] = hi;
            wl[kp * WP2 + m] = lo;
        }
        __syncthreads();   // W2 chunk (and, first pass, the hidden tile) visible
        if (co0 + 64 < C) load_w2(co0 + 64);
        float acc2[2][NT2][4];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < NT2; ++j) acc2[i][j][0] = acc2[i][j][1] = acc2[i][j][2] = acc2[i][j][3] = 0.f;
#pragma unroll 1
        for (int kb = 0; kb < HD / 16; ++kb) {      // one k16 step = 16 hidden channels = one tensor-core accumulation run
            const int ho = (kb * 8 + c) * RB_XSP + wn2 * (8 * NT2) + g;
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {        // one m tile at a time: 2 x NT2 x 4 run accumulators live instead of 4 x
                float c0[NT2][4], c1[NT2][4];
#pragma unroll
                for (int j = 0; j < NT2; ++j) {
                    c0[j][0] = c0[j][1] = c0[j][2] = c0[j][3] = 0.f;
                    c1[j][0] = c1[j][1] = c1[j][2] = c1[j][3] = 0.f;
                }
                const int m = wm2 * 32 + mt * 16 + g, kr = kb * 8;
                uint32_t ah[4], al[4];
                ah[0] = wh[(kr + c) * WP2 + m];     ah[1] = wh[(kr + c) * WP2 + m + 8];
                ah[2] = wh[(kr + c + 4) * WP2 + m]; ah[3] = wh[(kr + c + 4) * WP2 + m + 8];
                al[0] = wl[(kr + c) * WP2 + m];     al[1] = wl[(kr + c) * WP2 + m + 8];
                al[2] = wl[(kr + c + 4) * WP2 + m]; al[3] = wl[(kr + c + 4) * WP2 + m + 8];
#pragma unroll
                for (int nt = 0; nt < NT2; ++nt) {
                    const uint32_t bh0 = xh[ho + nt * 8], bh1 = xh[ho + 4 * RB_XSP + nt * 8];
                    const uint32_t bl0 = xl[ho + nt * 8], bl1 = xl[ho + 4 * RB_XSP + nt * 8];
                    mma_f16r(c0[nt], ah, bh0, bh1);
                    mma_f16r(c1[nt], ah, bl0, bl1);
                    mma_f16r(c1[nt], al, bh0, bh1);
                }
#pragma unroll
                for (int j = 0; j < NT2; ++j)
#pragma unroll
                    for (int e = 0; e < 4; ++e) acc2[mt][j][e] += fmaf(c1[j][e], LO, c0[j][e]);
            }
        }
        // the skip connection under this warp's output tile
        float2 xsk[2][2][NT2];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int hrow = 0; hrow < 2; ++hrow) {
                const int co = co0 + wm2 * 32 + mt * 16 + g + 8 * hrow;
                const float* __restrict__ xr = xb + (size_t)co * p.T;
#pragma unroll
                for (int nt = 0; nt < NT2; ++nt) {
                    const int t = t0 + wn2 * (8 * NT2) + nt * 8 + 2 * c;
                    if (pair_ok && t + 1 < p.T) xsk[mt][hrow][nt] = __ldg(reinterpret_cast<const float2*>(xr + t));
                    else xsk[mt][hrow][nt] = make_float2(t < p.T ? __ldg(xr + t) : 0.f, t + 1 < p.T ? __ldg(xr + t + 1) : 0.f);
                }
            }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int hrow = 0; hrow < 2; ++hrow) {
                const int co = co0 + wm2 * 32 + mt * 16 + g + 8 * hrow;
                const float bv = __ldg(p.b2 + co);
                float* yr = p.y + ((size_t)b * C + co) * p.T;
#pragma unroll
                for (int nt = 0; nt < NT2; ++nt) {
                    const int t = t0 + wn2 * (8 * NT2) + nt * 8 + 2 * c;
                    const float v0 = acc2[mt][nt][2 * hrow] + bv + xsk[mt][hrow][nt].x;
                    const float v1 = acc2[mt][nt][2 * hrow + 1] + bv + xsk[mt][hrow][nt].y;
                    if (pair_ok && t + 1 < p.T) {
                        *reinterpret_cast<float2*>(yr + t) = make_float2(v0, v1);
                    } else {
                        if (t < p.T) yr[t] = v0;
                        if (t + 1 < p.T) yr[t + 1] = v1;
                    }
                }
            }
    }
}

template <int HD, bool FLUSH>
static int launch_resblock_one(const ResblockParams& p, int batch, cudaStream_t s) {
    constexpr int C = 2 * HD, WP1 = HD + 8, WP2 = 72;
    constexpr int WHALF = (3 * RB_CH * WP1) > (HD * WP2) ? (3 * RB_CH * WP1) : (HD * WP2);
    const size_t smem = ((size_t)C * RB_XSP + 2 * (size_t)WHALF) * sizeof(float);
    ACB_CHECK_CUDA(cudaFuncSetAttribute(resblock_kernel<HD, FLUSH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(acb_ceil_div(p.T, RB_TB), batch);
    resblock_kernel<HD, FLUSH><<<grid, HD >= 128 ? 512 : 256, smem, s>>>(p);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

template <int HD, bool FLUSH>
static int launch_resblock_h2(const ResblockParams& p, int batch, cudaStream_t s) {
    constexpr int C = 2 * HD, WP1 = HD + 8, WP2 = 72, KP1 = 3 * RB_CH / 2;
    constexpr int WHALF = (KP1 * WP1) > ((HD / 2) * WP2) ? (KP1 * WP1) : ((HD / 2) * WP2);
    const size_t smem = ((size_t)C * RB_XSP + 2 * (size_t)WHALF) * sizeof(uint32_t);
    ACB_CHECK_CUDA(cudaFuncSetAttribute(resblock_h2_kernel<HD, FLUSH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(acb_ceil_div(p.T, RB_TB), batch);
    resblock_h2_kernel<HD, FLUSH><<<grid, HD >= 128 ? 512 : 256, smem, s>>>(p);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

extern "C" int acb_resblock_supported(int channels, int kernel, int dilation) {
    return (channels == 64 || channels == 128 || channels == 256) && kernel == 3 && dilation >= 1 && 2 * dilation <= RB_XSP - RB_TB;
}

extern "C" int acb_resblock(const float* x, const float* w1, const float* b1, const float* w2, const float* b2, float* y, int batch,
                            int channels, int t_len, int kernel, int dilation, int pad_left, int reflect, int exact, void* stream) {
    ACB_REQUIRE(x && w1 && b1 && w2 && b2 && y && x != y, "acb_resblock: null or aliased pointer");
    ACB_REQUIRE(acb_resblock_supported(channels, kernel, dilation), "acb_resblock: C=%d k=%d dilation=%d is not built", channels, kernel, dilation);
    ACB_REQUIRE(batch > 0 && batch <= 65535 && t_len > 0 && pad_left >= 0 && pad_left <= 2 * dilation, "acb_resblock: bad shape");
    ACB_REQUIRE(!reflect || t_len > 2 * dilation, "acb_resblock: reflect padding needs t_len > %d", 2 * dilation);
    ResblockParams p{x, w1, b1, w2, b2, y, t_len, dilation, pad_left, reflect};
    cudaStream_t s = (cudaStream_t)stream;
    {   // default: operands split into fp16 terms (resblock_h2_kernel); ACB_RESBLOCK_TF32=1 keeps the 3xTF32 kernel (A/B)
        const char* e = getenv("ACB_RESBLOCK_TF32");
        if (!(e && e[0] == '1')) {
            switch (channels) {
                case 64: return exact ? launch_resblock_h2<32, true>(p, batch, s) : launch_resblock_h2<32, false>(p, batch, s);
                case 128: return exact ? launch_resblock_h2<64, true>(p, batch, s) : launch_resblock_h2<64, false>(p, batch, s);
                default: return exact ? launch_resblock_h2<128, true>(p, batch, s) : launch_resblock_h2<128, false>(p, batch, s);
            }
        }
    }
    switch (channels) {
        case 64: return exact ? launch_resblock_one<32, true>(p, batch, s) : launch_resblock_one<32, false>(p, batch, s);
        case 128: return exact ? launch_resblock_one<64, true>(p, batch, s) : launch_resblock_one<64, false>(p, batch, s);
        default: return exact ? launch_resblock_one<128, true>(p, batch, s) : launch_resblock_one<128, false>(p, batch, s);
    }
}

// ------------------------------------------------------------------------------------------------
// conv1d on the tensor cores: wgmma.mma_async tf32 (m64nNk8) with the accumulator in registers, 3xTF32 split.
//   D[64 time steps][N output channels] += A[64][8] . B[N][8]^T   per instruction and warpgroup; the two warpgroups of the
//   CTA own time steps [0, 64) and [64, 128) of the tile
//   A = im2col rows of the staged input slab, B = weight rows, both K-major in the canonical 128-byte-swizzled layout
//       offset(row, k16B) = row * 128 B + ((k16B ^ (row % 8)) * 16 B)              (one 32-row reduction chunk = one 128-byte row)
// Per reduction chunk of 32 rows (r = channel x tap) every thread builds its im2col row (hi and lo tf32 parts) and a
// share of the weight tile, a proxy fence publishes them to the async proxy, each warpgroup issues 4 k-steps x 3 MMAs
// (lo*hi, hi*lo, hi*hi) and waits for them; the epilogue fuses bias + residual into the stores.
// ------------------------------------------------------------------------------------------------
constexpr int T5_M = 128, T5_RC = 32;

// TERMS = 2: x ~ hi + lo -> 3 MMAs per product (lo*hi, hi*lo, hi*hi).  (A 3-term / 6-MMA split was measured: identical
// end-to-end error, 1.43e-4 on the 32 kHz latents -- the residual is the tensor core's accumulate rounding, not the
// operand split -- so only the 2-term variant is built.)
constexpr int T5_SLAB_PT = 16;   // staged input elements per thread and chunk (<= 4096 per chunk)

template <int TERMS>
__device__ __forceinline__ void t5_split(float x, float (&out)[TERMS]) {
    float rem = x;
#pragma unroll
    for (int i = 0; i < TERMS; ++i) {
        out[i] = __uint_as_float(to_tf32(rem));
        rem -= out[i];
    }
}

template <int TERMS, int NW>   // NW = weight elements per thread and chunk = N * 32 / 256
__global__ void __launch_bounds__(256, NW >= 8 ? 1 : 2) conv1d_t5_kernel(ConvParams p, int xsp) {
    constexpr int N = NW * 8;
    extern __shared__ __align__(1024) unsigned char t5sm[];   // swizzled operand tiles are 1024-byte aligned
    // [A terms: TERMS x 16 KB][B terms: TERMS x N*128 B][slab][roff]
    float* a_t = reinterpret_cast<float*>(t5sm);
    float* b_t = a_t + TERMS * T5_M * T5_RC;
    float* xs = b_t + TERMS * N * T5_RC;
    int* roff = reinterpret_cast<int*>(xs + ((p.ci_chunk * xsp + 3) & ~3));   // keep 16-byte alignment behind the slab

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int t0 = blockIdx.x * T5_M, co0 = blockIdx.y * N, b = blockIdx.z;
    const float* xb = p.x + (size_t)b * p.c_in * p.t_in;

    // ---- chunk-invariant staging maps: where each of this thread's slab elements comes from (relative to the first
    //      channel of a chunk) and where it goes (phase-de-interleaved slab), computed once
    const int g0 = t0 * p.stride - p.pad_left;
    int src_off[T5_SLAB_PT], dcl[T5_SLAB_PT];   // dcl = slab destination | (channel-in-chunk << 24), -1 = no element
    const int n_slab = p.ci_chunk * p.span;
#pragma unroll
    for (int i = 0; i < T5_SLAB_PT; ++i) {
        const int e = tid + 256 * i;
        src_off[i] = -1; dcl[i] = -1;
        if (e < n_slab) {
            const int cl = e / p.span, j = e - cl * p.span;
            int g = g0 + j;
            if (p.reflect) {
                if (g < 0) g = -g;
                if (g >= p.t_virt) g = 2 * (p.t_virt - 1) - g;
            }
            dcl[i] = (cl * xsp + (p.stride == 1 ? j : (j % p.stride) * p.PL + j / p.stride)) | (cl << 24);
            if (g >= 0 && g < p.t_in) src_off[i] = cl * p.t_in + g;   // else: padding -> 0
        }
    }
    for (int r = tid; r < T5_RC; r += 256) {   // reduction row r = (channel, tap) -> slab offset (chunk-invariant too)
        const int cl = r / p.K, k = r - cl * p.K, kd = k * p.dil;
        roff[r] = cl < p.ci_chunk ? cl * xsp + (kd % p.stride) * p.PL + kd / p.stride : 0;
    }
    __syncthreads();

    // this warpgroup's 64 rows of A start 64 x 128 B into each A term
    const uint32_t a_s = smem_u32_(a_t) + (uint32_t)wg * (64u * 128u), b_s = smem_u32_(b_t);
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;

    float xr[T5_SLAB_PT], wr[NW];
    auto prefetch = [&](int ci0) {   // raw global values of one chunk into registers (no dependence on smem state)
        const int nci = min(p.ci_chunk, p.c_in - ci0), rc = nci * p.K;
        const float* xc = xb + (size_t)ci0 * p.t_in;
#pragma unroll
        for (int i = 0; i < T5_SLAB_PT; ++i)
            xr[i] = (src_off[i] >= 0 && (dcl[i] >> 24) < nci) ? __ldg(xc + src_off[i]) : 0.f;
#pragma unroll
        for (int i = 0; i < NW; ++i) {
            const int idx = tid + 256 * i, r = idx / N, cc = idx % N;
            wr[i] = (r < rc && co0 + cc < p.c_out) ? __ldg(p.w + ((size_t)ci0 * p.K + r) * p.c_out + co0 + cc) : 0.f;
        }
    };
    prefetch(0);

    for (int ci0 = 0; ci0 < p.c_in; ci0 += p.ci_chunk) {
        // (the previous chunk's MMAs have completed -- waited at the bottom -- so slab and tiles may be rewritten)
#pragma unroll
        for (int i = 0; i < T5_SLAB_PT; ++i)
            if (dcl[i] >= 0) xs[dcl[i] & 0xFFFFFF] = p.elu ? acb_elu(xr[i]) : xr[i];
#pragma unroll
        for (int i = 0; i < NW; ++i) {
            const int idx = tid + 256 * i, r = idx / N, cc = idx % N;
            float parts[TERMS];
            t5_split<TERMS>(wr[i], parts);
            const int o = cc * 32 + (((r >> 2) ^ (cc & 7)) << 2) + (r & 3);   // row cc (128 B), chunk r/4 at position (r/4) ^ (cc & 7), in floats
#pragma unroll
            for (int q = 0; q < TERMS; ++q) b_t[q * N * T5_RC + o] = parts[q];
        }
        if (ci0 + p.ci_chunk < p.c_in) prefetch(ci0 + p.ci_chunk);   // next chunk's global loads fly during build + MMA
        __syncthreads();   // slab ready
        {   // im2col tile A[t][r]: threads 0..127 own one time step each for r in [0,16), threads 128..255 for [16,32)
            const int t = tid & 127, rbase = (tid >> 7) * 16;
#pragma unroll
            for (int kc = 0; kc < 4; ++kc) {   // 16-byte k-chunks of 4 reduction rows
                float parts[4][TERMS];
#pragma unroll
                for (int e = 0; e < 4; ++e) t5_split<TERMS>(xs[roff[rbase + kc * 4 + e] + t], parts[e]);
                const int o = t * 32 + ((((rbase >> 2) + kc) ^ (t & 7)) << 2);   // row t (128 B), chunk at position chunk ^ (t & 7), in floats
#pragma unroll
                for (int q = 0; q < TERMS; ++q)
                    *reinterpret_cast<float4*>(a_t + q * T5_M * T5_RC + o) =
                        make_float4(parts[0][q], parts[1][q], parts[2][q], parts[3][q]);
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
        __syncthreads();
        wgmma_fence();
        wgmma_fence_regs(acc);
#pragma unroll
        for (int ks = 0; ks < T5_RC / 8; ++ks) {   // one instruction = 8 reduction rows = two 16-byte k-chunks
            uint64_t ad[TERMS], bd[TERMS];
#pragma unroll
            for (int q = 0; q < TERMS; ++q) {
                ad[q] = wgmma_desc_sw128(a_s + q * (T5_M * T5_RC * 4) + ks * 32);
                bd[q] = wgmma_desc_sw128(b_s + q * (N * T5_RC * 4) + ks * 32);
            }
            // smallest cross terms first; term index 0 = hi.  Keep products a_i * b_j with i + j < TERMS.
#pragma unroll
            for (int sum = TERMS - 1; sum >= 0; --sum)
#pragma unroll
                for (int i = 0; i <= sum; ++i) wgmma_tf32<N>(acc, ad[i], bd[sum - i], 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        __syncthreads();   // both warpgroups are done reading this chunk's tiles
    }
    {   // thread (warp w of the warpgroup, lane l): time steps 64 wg + 16 w + l / 4 (+ 8), channels 8 j + 2 (l % 4) (+ 1)
        const int tr = t0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
            const int t = tr + ((i >> 1) & 1) * 8, c = co0 + (i >> 2) * 8 + (lane & 3) * 2 + (i & 1);
            if (t >= p.t_out || c >= p.c_out) continue;
            if (p.tr_S == 0) {
                const size_t o = ((size_t)b * p.c_out + c) * p.t_out + t;
                float y = acc[i] + (p.bias ? p.bias[c] : 0.f);
                if (p.res) y += p.res[o];
                p.y[o] = y;
            } else {   // transposed conv: column n' = co*S + phase, output step = t*S + phase - trim
                const int cout = p.c_out / p.tr_S, co = c / p.tr_S, ph = c - co * p.tr_S, o = t * p.tr_S + ph - p.tr_trim;
                if (o >= 0 && o < p.tr_tout)
                    p.y[((size_t)b * cout + co) * p.tr_tout + o] = acc[i] + (p.bias ? p.bias[co] : 0.f);
            }
        }
    }
}

template <int TERMS, int NW>
static int launch_t5_one(const ConvParams& q, int xsp, int batch, cudaStream_t s) {
    constexpr int N = NW * 8;
    size_t smem = ((size_t)TERMS * T5_M * T5_RC + (size_t)TERMS * N * T5_RC + (size_t)((q.ci_chunk * xsp + 3) & ~3)) * sizeof(float) +
                  T5_RC * sizeof(int);
    ACB_REQUIRE(smem <= 200 * 1024, "acb_conv1d: tensor-core tile needs %zu B of shared memory", smem);
    ACB_CHECK_CUDA(cudaFuncSetAttribute(conv1d_t5_kernel<TERMS, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(acb_ceil_div(q.t_out, T5_M), acb_ceil_div(q.c_out, N), batch);
    conv1d_t5_kernel<TERMS, NW><<<grid, 256, smem, s>>>(q, xsp);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

static int launch_conv1d_t5(const ConvParams& p, int batch, cudaStream_t s) {
    ConvParams q = p;
    q.ci_chunk = max(1, min(p.c_in, T5_RC / p.K));
    q.span = (T5_M - 1) * p.stride + (p.K - 1) * p.dil + 1;
    q.PL = acb_ceil_div(q.span, p.stride);
    const int xsp = p.stride * q.PL;
    ACB_REQUIRE(q.ci_chunk * q.span <= 256 * T5_SLAB_PT, "acb_conv1d: tensor-core slab too large (%d elements)", q.ci_chunk * q.span);
    // N <= 128: the 64 x N accumulator of each warpgroup lives in registers (64 per thread at N = 128)
    if (p.c_out >= 128) return launch_t5_one<2, 16>(q, xsp, batch, s);
    if (p.c_out >= 64) return launch_t5_one<2, 8>(q, xsp, batch, s);
    return launch_t5_one<2, 4>(q, xsp, batch, s);
}

// ------------------------------------------------------------------------------------------------
// The encoder's kernel for k > 1 with >= 128 output channels (EncodecModel encoder_precision='fp32_tc'): raw input samples
// through a cp.async ring, the CTA persistent over tiles.
//
// conv1d_t6: implicit-GEMM convolution on wgmma WITHOUT an im2col tile, warp-specialised and double-buffered, with
// the tensor-core accumulator flushed into fp32 registers once per 8-channel group.  It answers two problems of
// conv1d_t5_kernel:
//   (1) t5 is BUILD-bound, not MMA-bound: per 32 reduction rows it writes a 128 x 32 im2col tile (every input sample
//       is split and stored once per tap).  Here the reduction index of one MMA is 8 consecutive INPUT CHANNELS at a
//       fixed tap, and the staged input slab is laid out [4-channel chunk][stride phase][time][4 channels], i.e. with
//       SBO = 128 B the 128 time rows of the A operand are linear at 16 B pitch: a tap is just a different START ADDRESS
//       of the shared-memory descriptor (phase plane (k*D) % S, row offset (k*D) / S).  Each input sample is split and
//       stored once per 8-channel group instead of once per tap (7-16x less build work).
//   (2) t5's error is the tensor core's truncating fp32 accumulate over up to 3 072 chained MMAs.  Here the chain is
//       3*K MMAs (one 8-channel group) into a fresh accumulator, which is then added to register accumulators with
//       round-to-nearest fp32 adds.
// Roles (384 threads): warpgroup 0 (warps 0-3) stages the input slab (ELU, reflect / zero padding, hi/lo tf32 split);
// warpgroups 1 and 2 issue the MMAs on time steps [0, 64) and [64, 128) of the tile and own those rows of the output, and
// thread 0 of warpgroup 1 streams the pre-split, pre-laid-out weight tiles with TMA bulk copies, refilling each weight stage as
// soon as both warpgroups have released it (a producer-side loader would block the slab staging behind that release).  Pipelines: slab x2 (a_full / a_empty), weight
// stage x2 (b_full / b_empty); every consumer warp arrives on the empty barriers once its MMAs have completed.
// Weights are packed by the host as w6[co_tile][cg][k][term(hi,lo)][c(2)][n(N)][4 channels]  (fp32 bits, tf32-exact).
// ------------------------------------------------------------------------------------------------
constexpr int T6_M = 128, T6_THREADS = 384, T6_MAXV = 20;

struct T6Params {
    const float* x; const float* w6; const float* bias; const float* res; float* y;
    int c_in, c_out, t_in, t_virt, t_out, K, S, D, pad_left, reflect, elu;
    int span, PL, n_cg, TB;   // slab length, rows per phase plane, 8-channel groups, taps per weight stage
    int t_tiles, n_co, n_tiles;   // persistent tile loop: tile -> (time tile, output-channel tile, item)
    int raw_vec;                  // slab vectors per staging thread in use (<= NV)
};

__device__ __forceinline__ void t6_mbar_init(uint64_t* b, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32_(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void t6_mbar_arrive(uint64_t* b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32_(b)) : "memory");
}
__device__ __forceinline__ void t6_mbar_expect_tx(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32_(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void t6_mbar_wait(uint64_t* b, uint32_t parity) {
    uint32_t ok = 0;
    do {
        asm volatile("{\n .reg .pred q;\n mbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\n selp.u32 %0, 1, 0, q;\n}"
                     : "=r"(ok) : "r"(smem_u32_(b)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void t6_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32_(dst)), "l"(src), "r"(bytes), "r"(smem_u32_(bar)) : "memory");
}

// shared-memory layout (bytes), shared by kernel and launcher
struct T6Smem { int slab_term, slab_stage, b_tap, b_stage, slab, btile, bars, raw, raw_stage, total; };
// raw_vec = slab vectors per staging thread actually used (ceil(2 span / 128)), raw_depth = channel groups of raw input in flight per CTA
// (cp.async ring; 0 = the register-prefetch kernel)
__host__ __device__ inline T6Smem t6_smem(int N, int S, int PL, int TB, int raw_vec, int raw_depth) {
    T6Smem L;
    L.slab_term = 2 * S * PL * 16;          // [c(2)][phase][row][4 floats]
    L.slab_stage = 2 * L.slab_term;         // hi, lo
    L.b_tap = 2 * 2 * N * 16;               // [term][c(2)][n][4 floats]
    L.b_stage = TB * L.b_tap;
    L.slab = 0;
    L.btile = 2 * L.slab_stage;
    L.bars = L.btile + 2 * L.b_stage;
    L.raw = L.bars + 8 * 8;                 // [DEPTH][NV][4 channels][128 threads] raw samples (NV <= 12 only)
    L.raw_stage = raw_vec * 4 * 128 * 4;
    L.total = L.raw + raw_depth * L.raw_stage;
    return L;
}

// NV = slab vectors per staging thread (4 / 12 / 20): the maps and the prefetched raw samples live in registers; 12 warps cap the
// kernel at 168 registers per thread.
template <int N, int NV, int DEPTH>   // DEPTH: cp.async ring depth (0: register prefetch)
__global__ void __launch_bounds__(T6_THREADS, 1) conv1d_t6_kernel(T6Params p) {
    extern __shared__ __align__(128) unsigned char t6sm[];
    const T6Smem L = t6_smem(N, p.S, p.PL, p.TB, p.raw_vec, DEPTH);
    uint64_t* bars = reinterpret_cast<uint64_t*>(t6sm + L.bars);
    uint64_t* a_full = bars;          // [2] slab staged            (1 arrival: elected producer)
    uint64_t* a_empty = bars + 2;     // [2] slab consumed          (8 arrivals: one per consumer warp)
    uint64_t* b_full = bars + 4;      // [2] weight stage landed    (1 arrival + TMA bytes)
    uint64_t* b_empty = bars + 6;     // [2] weight stage consumed  (8 arrivals: one per consumer warp)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wgi = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warpgroup index, provably warp-uniform (keeps the MMAs pipelined)
    // PERSISTENT over tiles (one CTA per SM fits: 131 KB of shared memory): tile = blockIdx.x, += gridDim.x.  Every
    // role walks the same tile sequence with running group / stage counters, so the mbarrier pipelines simply continue across tiles:
    // the staging warps fill the next tile's first slabs while the consumers still work on (and store) the previous tile.
    const int nstage_b = (p.K + p.TB - 1) / p.TB;   // weight stages per channel group

    if (tid == 0) {
        for (int i = 0; i < 2; ++i) {
            t6_mbar_init(a_full + i, 1); t6_mbar_init(a_empty + i, 8);
            t6_mbar_init(b_full + i, 1); t6_mbar_init(b_empty + i, 8);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wgi == 0) {
        // ================= producers: stage the 8-channel slab of every channel group =================
        // chunk-invariant maps: this thread's (time j, 4-channel chunk c) vectors -> source index / destination
        const int nvec = 2 * p.span;
        int src[NV], dst[NV], jj[NV];   // src: input index or -1 (padding); dst: byte offset inside one term's slab or -1; jj: slab step
#pragma unroll
        for (int i = 0; i < NV; ++i) {   // tile-invariant part of the map (the divisions)
            const int e = tid + 128 * i;
            dst[i] = -1; jj[i] = 0;
            if (e < nvec) {
                const int c = e / p.span, j = e - c * p.span;
                dst[i] = (((c * p.S + (j % p.S)) * p.PL + j / p.S) * 16) | (c << 30);
                jj[i] = j;
            }
        }
        int G = 0;   // running channel-group counter (slab buffer = G & 1)
        if constexpr (DEPTH > 0) {
        // ---- raw samples through a cp.async ring, DEPTH channel groups deep.  The input streams from HBM (every sample is used by
        //      two tiles at most): one register batch per group in flight leaves too few bytes outstanding to cover HBM latency.
        //      The ring keeps 3-4 groups (50-70 KB) in flight, costs no registers, and runs across tile boundaries.
        float* rawsm = reinterpret_cast<float*>(t6sm + L.raw);
        const int raw_stage = p.raw_vec * 4 * 128;
        int itile = blockIdx.x, icg = 0, islot = 0;
        auto issue = [&]() {
            if (itile < p.n_tiles) {
                const int it0 = (itile % p.t_tiles) * T6_M, ib = itile / (p.t_tiles * p.n_co);
                const int ig0 = it0 * p.S - p.pad_left;
                const float* ixb = p.x + ((size_t)ib * p.c_in + (size_t)icg * 8) * p.t_in;
                const uint32_t rs = smem_u32_(rawsm + islot * raw_stage + tid);
#pragma unroll
                for (int i = 0; i < NV; ++i) {
                    if (dst[i] >= 0) {
                        int g = ig0 + jj[i];
                        if (p.reflect) {
                            if (g < 0) g = -g;
                            if (g >= p.t_virt) g = 2 * (p.t_virt - 1) - g;
                        }
                        const bool ok = g >= 0 && g < p.t_in;
                        const float* sp = ixb + (size_t)(((dst[i] >> 30) & 1) * 4) * p.t_in + (ok ? g : 0);
                        const uint32_t nbytes = ok ? 4u : 0u;   // 0: zero-fill (padding)
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(rs + (uint32_t)((i * 4 + q) * 128 * 4)),
                                         "l"(sp + (size_t)q * p.t_in), "r"(nbytes) : "memory");
                    }
                }
                if (++icg == p.n_cg) { icg = 0; itile += gridDim.x; }
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            islot = islot + 1 == DEPTH ? 0 : islot + 1;
        };
#pragma unroll 1
        for (int d = 0; d < DEPTH; ++d) issue();
        int cslot = 0;
        for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x)
        for (int cg = 0; cg < p.n_cg; ++cg, ++G) {
            const int st = G & 1;
            asm volatile("cp.async.wait_group %0;" ::"n"(DEPTH - 1) : "memory");   // this thread's copies of the oldest group have landed
            t6_mbar_wait(a_empty + st, ((G >> 1) & 1) ^ 1);   // first use of each buffer passes at once
            unsigned char* hi = t6sm + L.slab + st * L.slab_stage;
            unsigned char* lo = hi + L.slab_term;
            const float* rw = rawsm + cslot * raw_stage + tid;
#pragma unroll
            for (int i = 0; i < NV; ++i) {
                if (dst[i] < 0) continue;
                const int off = dst[i] & 0x3FFFFFFF;
                float h[4], l[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float r = rw[(i * 4 + q) * 128];
                    const float v = p.elu ? acb_elu(r) : r;
                    h[q] = __uint_as_float(to_tf32(v));
                    l[q] = __uint_as_float(to_tf32(v - h[q]));
                }
                *reinterpret_cast<float4*>(hi + off) = make_float4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<float4*>(lo + off) = make_float4(l[0], l[1], l[2], l[3]);
            }
            issue();   // refill the slot just consumed (islot == cslot here)
            cslot = cslot + 1 == DEPTH ? 0 : cslot + 1;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
            asm volatile("bar.sync 1, 128;" ::: "memory");                 // the four producer warps
            if (tid == 0) t6_mbar_arrive(a_full + st);
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        } else {
        for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const int t0 = (tile % p.t_tiles) * T6_M, b = tile / (p.t_tiles * p.n_co);
        const int g0 = t0 * p.S - p.pad_left;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            int g = g0 + jj[i];
            if (p.reflect) {
                if (g < 0) g = -g;
                if (g >= p.t_virt) g = 2 * (p.t_virt - 1) - g;
            }
            src[i] = (dst[i] >= 0 && g >= 0 && g < p.t_in) ? g : -1;
        }
        const float* xb = p.x + (size_t)b * p.c_in * p.t_in;
        // The raw samples of a channel group are requested as one batch into registers and consumed afterwards (loading, ELU-ing and
        // storing vector by vector makes every vector a dependent L2 round trip).  The next group's batch is requested
        // before this group is published, so its round trip overlaps the fence / barrier / wait for the buffer.
        float raw[NV][4];
        auto fetch = [&](int cg) {
#pragma unroll
            for (int i = 0; i < NV; ++i) {
                const int c = (dst[i] >> 30) & 1;
                const float* xc = xb + (size_t)(cg * 8 + c * 4) * p.t_in;
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    raw[i][q] = (dst[i] >= 0 && src[i] >= 0) ? __ldg(xc + (size_t)q * p.t_in + src[i]) : 0.f;
            }
        };
        fetch(0);
        for (int cg = 0; cg < p.n_cg; ++cg, ++G) {
            const int st = G & 1;
            t6_mbar_wait(a_empty + st, ((G >> 1) & 1) ^ 1);   // first use of each buffer passes at once
            unsigned char* hi = t6sm + L.slab + st * L.slab_stage;
            unsigned char* lo = hi + L.slab_term;
#pragma unroll
            for (int i = 0; i < NV; ++i) {
                if (dst[i] < 0) continue;
                const int off = dst[i] & 0x3FFFFFFF;
                float h[4], l[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float v = p.elu ? acb_elu(raw[i][q]) : raw[i][q];
                    h[q] = __uint_as_float(to_tf32(v));
                    l[q] = __uint_as_float(to_tf32(v - h[q]));
                }
                *reinterpret_cast<float4*>(hi + off) = make_float4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<float4*>(lo + off) = make_float4(l[0], l[1], l[2], l[3]);
            }
            if (cg + 1 < p.n_cg) fetch(cg + 1);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
            asm volatile("bar.sync 1, 128;" ::: "memory");                 // the four producer warps
            if (tid == 0) t6_mbar_arrive(a_full + st);
        }
        }   // tiles
        }   // register path (NV > 12)
    } else {
        // ================= consumers: warpgroup wg issues the MMAs of time steps [64 wg, +64) and owns those output rows =================
        const int wg = wgi - 1;
        const uint32_t lbo_a = (uint32_t)(p.S * p.PL * 16), lbo_b = (uint32_t)N * 16u;
        const uint32_t slab_s = smem_u32_(t6sm + L.slab) + (uint32_t)wg * (64u * 16u), btile_s = smem_u32_(t6sm + L.btile);
        float acc[N / 2], accr[N / 2];
        int it = 0, G = 0;
        // weight loader (thread 128): a cursor over the CTA's weight-stage sequence (tile, channel group, tap block)
        const bool loader = tid == 128;
        int ltile = blockIdx.x, lcg = 0, lsb = 0, lit = 0;
        auto load_next = [&]() {
            if (ltile >= p.n_tiles) return;
            const int bs = lit & 1, k0 = lsb * p.TB, ntap = min(p.TB, p.K - k0);
            t6_mbar_wait(b_empty + bs, ((lit >> 1) & 1) ^ 1);   // both warpgroups are done with the stage's previous use
            const unsigned char* wbase = reinterpret_cast<const unsigned char*>(p.w6) +
                                         (size_t)((ltile / p.t_tiles) % p.n_co) * p.n_cg * p.K * L.b_tap;
            const uint32_t bytes = (uint32_t)ntap * (uint32_t)L.b_tap;
            t6_mbar_expect_tx(b_full + bs, bytes);
            t6_bulk_g2s(t6sm + L.btile + bs * L.b_stage, wbase + ((size_t)lcg * p.K + k0) * L.b_tap, bytes, b_full + bs);
            ++lit;
            if (++lsb == nstage_b) { lsb = 0; if (++lcg == p.n_cg) { lcg = 0; ltile += gridDim.x; } }
        };
        if (loader) { load_next(); load_next(); }
        __syncwarp();
        for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
            const int t0 = (tile % p.t_tiles) * T6_M, co0 = ((tile / p.t_tiles) % p.n_co) * N, b = tile / (p.t_tiles * p.n_co);
#pragma unroll
            for (int j = 0; j < N / 2; ++j) accr[j] = 0.f;
            for (int cg = 0; cg < p.n_cg; ++cg, ++G) {
                const int st = G & 1;
                t6_mbar_wait(a_full + st, (G >> 1) & 1);
                uint32_t scale_d = 0;   // the first MMA of a channel group overwrites the accumulator
                for (int sb = 0; sb < nstage_b; ++sb, ++it) {
                    const int bs = it & 1, k0 = sb * p.TB, ntap = min(p.TB, p.K - k0);
                    t6_mbar_wait(b_full + bs, (it >> 1) & 1);
                    wgmma_fence();
                    wgmma_fence_regs(acc);
                    for (int kk = 0; kk < ntap; ++kk) {
                        const int kd = (k0 + kk) * p.D;
                        const uint32_t a_off = (uint32_t)(((kd % p.S) * p.PL + kd / p.S) * 16);
                        const uint64_t a_hi = wgmma_desc(slab_s + st * L.slab_stage + a_off, lbo_a, 128);
                        const uint64_t a_lo = wgmma_desc(slab_s + st * L.slab_stage + L.slab_term + a_off, lbo_a, 128);
                        const uint32_t bt = btile_s + bs * L.b_stage + kk * L.b_tap;
                        const uint64_t b_hi = wgmma_desc(bt, lbo_b, 128), b_lo = wgmma_desc(bt + 2 * N * 16, lbo_b, 128);
                        wgmma_tf32<N>(acc, a_lo, b_hi, scale_d);   // small cross terms first
                        wgmma_tf32<N>(acc, a_hi, b_lo, 1u);
                        wgmma_tf32<N>(acc, a_hi, b_hi, 1u);
                        scale_d = 1u;
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_regs(acc);
                    __syncwarp();
                    if (lane == 0) t6_mbar_arrive(b_empty + bs);   // the weight stage may be overwritten
                    if (loader) load_next();                        // ... with the stage two ahead
                    __syncwarp();
                }
                if (lane == 0) t6_mbar_arrive(a_empty + st);       // ... and so may the slab
#pragma unroll
                for (int j = 0; j < N / 2; ++j) accr[j] += acc[j];  // round-to-nearest fp32 adds
            }
            // thread (warp w of the warpgroup, lane l): time steps 64 wg + 16 w + l / 4 (+ 8), channels 8 j + 2 (l % 4) (+ 1)
            const int tr = t0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
            for (int j = 0; j < N / 2; ++j) {
                const int t = tr + ((j >> 1) & 1) * 8, co = co0 + (j >> 2) * 8 + (lane & 3) * 2 + (j & 1);
                if (t < p.t_out && co < p.c_out) {
                    const size_t o = ((size_t)b * p.c_out + co) * p.t_out + t;
                    float yv = accr[j] + (p.bias ? p.bias[co] : 0.f);
                    if (p.res) yv += p.res[o];
                    p.y[o] = yv;
                }
            }
        }   // tiles
    }
}

template <int N, int NV, int DEPTH>
static int launch_t6_one(const T6Params& q, int batch, cudaStream_t s) {
    const T6Smem L = t6_smem(N, q.S, q.PL, q.TB, q.raw_vec, DEPTH);
    ACB_REQUIRE(L.total <= 227 * 1024, "acb_conv1d_t6: tile needs %d B of shared memory", L.total);
    ACB_CHECK_CUDA(cudaFuncSetAttribute(conv1d_t6_kernel<N, NV, DEPTH>, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total));
    T6Params r = q;
    r.t_tiles = acb_ceil_div(q.t_out, T6_M); r.n_co = q.c_out / N; r.n_tiles = r.t_tiles * r.n_co * batch;
    int dev = 0, sms = 0;
    ACB_CHECK_CUDA(cudaGetDevice(&dev));
    ACB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    conv1d_t6_kernel<N, NV, DEPTH><<<dim3(min(r.n_tiles, sms)), T6_THREADS, (size_t)L.total, s>>>(r);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

extern "C" int acb_conv1d_t6_tile(int c_out) { return c_out % 128 == 0 ? 128 : (c_out % 64 == 0 ? 64 : 0); }

extern "C" int acb_conv1d_t6(const float* x, const float* w6, const float* bias, const float* residual, float* y, int batch,
                             int c_in, int c_out, int t_in, int t_virtual, int t_out, int kernel, int stride, int dilation,
                             int pad_left, int reflect, int elu_in, void* stream) {
    ACB_REQUIRE(x && w6 && y, "acb_conv1d_t6: null pointer");
    ACB_REQUIRE(batch > 0 && batch <= 65535 && c_in > 0 && c_out > 0 && t_in > 0 && t_out > 0, "acb_conv1d_t6: bad shape");
    ACB_REQUIRE(kernel >= 1 && kernel <= 64 && stride >= 1 && dilation >= 1 && pad_left >= 0 && t_virtual >= t_in, "acb_conv1d_t6: bad taps");
    ACB_REQUIRE(c_in % 8 == 0, "acb_conv1d_t6: c_in %d is not a multiple of 8 (one MMA reduces over 8 channels)", c_in);
    const int N = acb_conv1d_t6_tile(c_out);
    ACB_REQUIRE(N != 0, "acb_conv1d_t6: c_out %d is not a multiple of 64", c_out);
    T6Params q{x, w6, bias, residual, y, c_in, c_out, t_in, t_virtual, t_out, kernel, stride, dilation, pad_left, reflect, elu_in,
               0, 0, c_in / 8, 0};
    q.span = (T6_M - 1) * stride + (kernel - 1) * dilation + 1;
    q.PL = acb_ceil_div(q.span, stride);
    q.TB = kernel < 4 ? kernel : 4;
    ACB_REQUIRE(2 * q.span <= 128 * T6_MAXV, "acb_conv1d_t6: slab too long (%d samples per channel)", q.span);
    cudaStream_t s = (cudaStream_t)stream;
    const int nv = acb_ceil_div(2 * q.span, 128);
    q.raw_vec = nv;
    // cp.async ring of raw samples, 4 or 3 channel groups deep, where it fits next to the slab and weight stages (227 KB); else the
    // register-prefetch kernel (long slabs x wide strides, e.g. k = 16, stride 8)
    const int lim = 227 * 1024;
    const int depth = nv > 12 ? 0 : (t6_smem(N, q.S, q.PL, q.TB, nv, 4).total <= lim ? 4 : (t6_smem(N, q.S, q.PL, q.TB, nv, 3).total <= lim ? 3 : 0));
#define ACB_T6_LAUNCH(NN)                                                                                             \
    do {                                                                                                              \
        if (depth == 0) return launch_t6_one<NN, 20, 0>(q, batch, s);                                                 \
        if (nv <= 4) return depth == 4 ? launch_t6_one<NN, 4, 4>(q, batch, s) : launch_t6_one<NN, 4, 3>(q, batch, s); \
        return depth == 4 ? launch_t6_one<NN, 12, 4>(q, batch, s) : launch_t6_one<NN, 12, 3>(q, batch, s);            \
    } while (0)
    if (N == 128) ACB_T6_LAUNCH(128);
    ACB_T6_LAUNCH(64);
#undef ACB_T6_LAUNCH
}

// Few output channels (the decoder's last conv, Cout = audio channels): a thread owns 4 consecutive output steps of
// every output channel and slides a register window over the taps, so the kernel is a pure stream over x.
constexpr int SC_MAXCO = 4, SC_TILE = 1024;
struct SmallCoParams {
    const float* x; const float* w; const float* bias; const float* res; float* y;
    int c_in, c_out, t_in, t_virt, t_out, K, pad_left, reflect, elu, ci_chunk;
};
template <int KT>
__global__ void __launch_bounds__(256) conv1d_small_cout_kernel(SmallCoParams p) {
    extern __shared__ float smem[];
    constexpr int span = SC_TILE + KT - 1;
    constexpr int pitch = SC_TILE + 12;            // row pitch: multiple of 4 floats so the window loads are LDS.128
    static_assert(KT + 3 <= 12, "window of 3 float4");
    float* xs = smem;                              // [ci_chunk][pitch]
    float* ws = xs + p.ci_chunk * pitch;           // [ci_chunk][KT][SC_MAXCO]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int t0 = blockIdx.x * SC_TILE, b = blockIdx.y;
    const float* xb = p.x + (size_t)b * p.c_in * p.t_in;
    float acc[SC_MAXCO][4];
#pragma unroll
    for (int c = 0; c < SC_MAXCO; ++c) acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f;
    const int g0 = t0 - p.pad_left;
    for (int ci0 = 0; ci0 < p.c_in; ci0 += p.ci_chunk) {
        const int nci = min(p.ci_chunk, p.c_in - ci0);
        __syncthreads();
        for (int cl = warp; cl < nci; cl += 8) {
            const float* xrow = xb + (size_t)(ci0 + cl) * p.t_in;
            stage_span(xs + cl * pitch, xrow, g0, 1, span, pitch, p.t_in, p.t_virt, p.reflect, p.elu, lane);
        }
        for (int idx = tid; idx < nci * KT * SC_MAXCO; idx += 256) {
            const int c = idx % SC_MAXCO, rk = idx / SC_MAXCO;   // rk = cl*KT + k
            ws[idx] = c < p.c_out ? p.w[((size_t)ci0 * KT + rk) * p.c_out + c] : 0.f;
        }
        __syncthreads();
        for (int cl = 0; cl < nci; ++cl) {
            float xw[12];
            const float4* xr4 = reinterpret_cast<const float4*>(xs + cl * pitch + tid * 4);
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const float4 v4 = xr4[i];
                xw[4 * i] = v4.x; xw[4 * i + 1] = v4.y; xw[4 * i + 2] = v4.z; xw[4 * i + 3] = v4.w;
            }
#pragma unroll
            for (int k = 0; k < KT; ++k) {
                const float4 wv = *reinterpret_cast<const float4*>(ws + (cl * KT + k) * SC_MAXCO);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    acc[0][j] = fmaf(wv.x, xw[k + j], acc[0][j]);
                    acc[1][j] = fmaf(wv.y, xw[k + j], acc[1][j]);
                    acc[2][j] = fmaf(wv.z, xw[k + j], acc[2][j]);
                    acc[3][j] = fmaf(wv.w, xw[k + j], acc[3][j]);
                }
            }
        }
    }
    for (int c = 0; c < p.c_out; ++c) {
        const float bv = p.bias ? p.bias[c] : 0.f;
        const size_t row = ((size_t)b * p.c_out + c) * p.t_out;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int t = t0 + tid * 4 + j;
            if (t < p.t_out) {
                float v = (c == 0 ? acc[0][j] : c == 1 ? acc[1][j] : c == 2 ? acc[2][j] : acc[3][j]) + bv;
                if (p.res) v += p.res[row + t];
                p.y[row + t] = v;
            }
        }
    }
}

template <int KT>
static int launch_small_cout(const SmallCoParams& p, int batch, cudaStream_t s) {
    SmallCoParams q = p;
    q.ci_chunk = min(p.c_in, 8);
    size_t smem = ((size_t)q.ci_chunk * (SC_TILE + 12) + (size_t)q.ci_chunk * KT * SC_MAXCO) * sizeof(float);
    dim3 grid(acb_ceil_div(p.t_out, SC_TILE), batch);
    conv1d_small_cout_kernel<KT><<<grid, 256, smem, s>>>(q);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

extern "C" int acb_conv1d(const float* x, const float* w_packed, const float* bias, const float* residual, float* y,
                          int batch, int c_in, int c_out, int t_in, int t_virtual, int t_out, int kernel, int stride,
                          int dilation, int pad_left, int reflect, int elu_in, int precision, void* stream) {
    ACB_REQUIRE(x && w_packed && y, "acb_conv1d: null pointer");
    ACB_REQUIRE(batch > 0 && c_in > 0 && c_out > 0 && t_in > 0 && t_out > 0, "acb_conv1d: empty shape");
    ACB_REQUIRE(kernel >= 1 && kernel <= 64 && stride >= 1 && dilation >= 1 && pad_left >= 0, "acb_conv1d: bad taps");
    ACB_REQUIRE(t_virtual >= t_in, "acb_conv1d: t_virtual < t_in");
    ACB_REQUIRE(batch <= 65535, "acb_conv1d: batch > 65535");
    ConvParams p{x, w_packed, bias, residual, y, c_in, c_out, t_in, t_virtual, t_out, kernel, stride, dilation,
                 pad_left, reflect, elu_in, 0, 0, 0, 0, 0, 0};
    cudaStream_t s = (cudaStream_t)stream;
    if (c_out <= SC_MAXCO && stride == 1 && dilation == 1 && (kernel == 7 || kernel == 3)) {
        SmallCoParams q{x, w_packed, bias, residual, y, c_in, c_out, t_in, t_virtual, t_out, kernel, pad_left, reflect, elu_in, 0};
        return kernel == 7 ? launch_small_cout<7>(q, batch, s) : launch_small_cout<3>(q, batch, s);
    }
    ACB_REQUIRE(precision >= ACB_CONV_FP32 && precision <= ACB_CONV_TF32X3_MMASYNC, "acb_conv1d: unknown precision %d", precision);
    if ((precision == ACB_CONV_TF32X3 || precision == ACB_CONV_TF32X3_MMASYNC) && c_out >= 32 && c_in * kernel >= 16 &&
        kernel <= T5_RC) {
        // the tensor-core kernel pays a fixed im2col-tile build per 32 reduction rows: it wins once the tile has >= 128 output channels
        // to amortise it over; narrower layers go to the mma.sync kernel
        if (precision == ACB_CONV_TF32X3 && c_out >= 128 && c_in * kernel >= 128) return launch_conv1d_t5(p, batch, s);
        return launch_conv1d_tc(p, batch, s);
    }
    const bool wide = t_out >= 2048;   // 8 output steps per thread once there is enough time axis to fill the tile
    if (c_out >= 64) return wide ? launch_conv1d<8, 8>(p, batch, s) : launch_conv1d<8, 4>(p, batch, s);
    if (c_out >= 32) return wide ? launch_conv1d<4, 8>(p, batch, s) : launch_conv1d<4, 4>(p, batch, s);
    if (c_out >= 16) return launch_conv1d<2, 4>(p, batch, s);
    return launch_conv1d<1, 4>(p, batch, s);
}

// ------------------------------------------------------------------------------------------------
// transposed conv1d (kernel = 2*stride) + trim, as S interleaved 2-tap convolutions: lane = input step ti,
// every thread produces the S consecutive outputs u = ti*S + p for CPT channels, so x is read once per
// input channel and reused over all phases.
// ------------------------------------------------------------------------------------------------
struct ConvTrParams {
    const float* x; const float* w; const float* bias; float* y;
    int c_in, c_out, t_in, t_out, trim_left, elu, ci_chunk;
};

template <int S, int CPT>
__global__ void __launch_bounds__(256) convtr1d_kernel(ConvTrParams p) {
    constexpr int K = 2 * S, BM = 8 * CPT;
    extern __shared__ float smem[];
    float* ws = smem;                        // [ci_chunk][K][BM]
    float* xs = ws + p.ci_chunk * K * BM;    // [ci_chunk][33]: slot l+1 <-> ti0+l, slot 0 <-> ti0-1

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ti0 = blockIdx.x * 32, co0 = blockIdx.y * BM, b = blockIdx.z;
    const float* xb = p.x + (size_t)b * p.c_in * p.t_in;

    float acc[CPT][S];
#pragma unroll
    for (int i = 0; i < CPT; ++i)
#pragma unroll
        for (int q = 0; q < S; ++q) acc[i][q] = 0.f;

    for (int ci0 = 0; ci0 < p.c_in; ci0 += p.ci_chunk) {
        const int nci = min(p.ci_chunk, p.c_in - ci0);
        __syncthreads();
        for (int idx = tid; idx < nci * K * BM; idx += 256) {
            int r = idx / BM, c = idx - r * BM;
            ws[idx] = (co0 + c < p.c_out) ? p.w[((size_t)ci0 * K + r) * p.c_out + co0 + c] : 0.f;
        }
        for (int idx = tid; idx < nci * 33; idx += 256) {
            int cl = idx / 33, l = idx - cl * 33;
            int ti = ti0 + l - 1;
            float v = (ti >= 0 && ti < p.t_in) ? xb[(size_t)(ci0 + cl) * p.t_in + ti] : 0.f;
            xs[idx] = p.elu ? acb_elu(v) : v;
        }
        __syncthreads();
        for (int cl = 0; cl < nci; ++cl) {
            const float xa = xs[cl * 33 + lane + 1], xp = xs[cl * 33 + lane];
            const float* wc = ws + cl * K * BM + warp * CPT;
#pragma unroll
            for (int q = 0; q < S; ++q) {
#pragma unroll
                for (int i = 0; i < CPT; ++i) {
                    acc[i][q] = fmaf(xa, wc[q * BM + i], acc[i][q]);
                    acc[i][q] = fmaf(xp, wc[(q + S) * BM + i], acc[i][q]);
                }
            }
        }
    }
    const int ti = ti0 + lane;
#pragma unroll
    for (int i = 0; i < CPT; ++i) {
        int co = co0 + warp * CPT + i;
        if (co >= p.c_out) continue;
        float bv = p.bias ? p.bias[co] : 0.f;
        size_t row = ((size_t)b * p.c_out + co) * p.t_out;
#pragma unroll
        for (int q = 0; q < S; ++q) {
            int o = ti * S + q - p.trim_left;
            if (o >= 0 && o < p.t_out) p.y[row + o] = acc[i][q] + bv;
        }
    }
}

template <int S>
static int launch_convtr(const ConvTrParams& p, int batch, cudaStream_t s) {
    constexpr int CPT = (S >= 8) ? 4 : 8, BM = 8 * CPT, K = 2 * S;
    ConvTrParams q = p;
    q.ci_chunk = max(1, min(p.c_in, 64 / K));
    size_t smem = ((size_t)q.ci_chunk * K * BM + (size_t)q.ci_chunk * 33) * sizeof(float);
    int n_ti = acb_ceil_div(p.t_out + p.trim_left, S);
    dim3 grid(acb_ceil_div(n_ti, 32), acb_ceil_div(p.c_out, BM), batch);
    convtr1d_kernel<S, CPT><<<grid, 256, smem, s>>>(q);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

extern "C" int acb_convtr1d(const float* x, const float* w_packed, const float* w_gemm, const float* bias, float* y, int batch,
                            int c_in, int c_out, int t_in, int t_out, int kernel, int stride, int trim_left, int elu_in,
                            int precision, void* stream) {
    ACB_REQUIRE(x && w_packed && y, "acb_convtr1d: null pointer");
    ACB_REQUIRE(batch > 0 && batch <= 65535 && c_in > 0 && c_out > 0 && t_in > 0 && t_out > 0, "acb_convtr1d: bad shape");
    ACB_REQUIRE(kernel == 2 * stride, "acb_convtr1d: only kernel == 2*stride is built (got k=%d s=%d)", kernel, stride);
    ACB_REQUIRE(trim_left >= 0 && t_out + trim_left <= (t_in + 1) * stride, "acb_convtr1d: trim out of range");
    ACB_REQUIRE(precision >= ACB_CONV_FP32 && precision <= ACB_CONV_TF32X3_MMASYNC, "acb_convtr1d: unknown precision %d", precision);
    cudaStream_t s = (cudaStream_t)stream;
    if (precision == ACB_CONV_TF32X3 && w_gemm && c_out * stride >= 128 && c_in >= 64) {
        // y[co][ti*S + ph - trim] = sum_{ci} x[ci][ti] w[ci][ph][co] + x[ci][ti-1] w[ci][ph+S][co]: a GEMM over 2-tap im2col
        // rows r = (ci, k) (k = 0: x[ti-1], k = 1: x[ti]) and virtual channels n' = co*S + ph; w_gemm is [2*Cin][Cout*S]
        const int n_ti = acb_ceil_div(t_out + trim_left, stride);
        ConvParams p{x, w_gemm, bias, nullptr, y, c_in, c_out * stride, t_in, t_in, n_ti, 2, 1, 1, 1, 0, elu_in, 0, 0, 0,
                     stride, trim_left, t_out};
        return launch_conv1d_t5(p, batch, s);
    }
    ConvTrParams p{x, w_packed, bias, y, c_in, c_out, t_in, t_out, trim_left, elu_in, 0};
    switch (stride) {
        case 2: return launch_convtr<2>(p, batch, s);
        case 3: return launch_convtr<3>(p, batch, s);
        case 4: return launch_convtr<4>(p, batch, s);
        case 5: return launch_convtr<5>(p, batch, s);
        case 8: return launch_convtr<8>(p, batch, s);
    }
    acb_set_error("acb_convtr1d: stride %d not built (2,3,4,5,8)", stride);
    return ACB_ERR_UNSUPPORTED;
}

// ------------------------------------------------------------------------------------------------
// LSTM recurrence: one persistent cooperative kernel for all T steps.  CTA c owns hidden units
// [c*U, (c+1)*U) i.e. 4U rows of W_hh, held in shared memory for the whole sequence; per step it reads
// h_{t-1} (all units) from L2, computes its 4U x B gate pre-activations, applies the cell update for its
// units and publishes h_t; a grid-wide barrier separates the steps.
// ------------------------------------------------------------------------------------------------
struct LstmParams {
    const float* gx; const float* whh; const float* skip; float* y; float* hbuf; unsigned* bar;
    int B, H, T, U;
};

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

constexpr int LSTM_BC = 16;  // batch items per matvec pass

__global__ void __launch_bounds__(256) lstm_kernel(LstmParams p) {
    extern __shared__ float smem[];
    const int H = p.H, U = p.U, R = 4 * U;
    float* wsm = smem;                      // [R][H]
    float* hs = wsm + (size_t)R * H;        // [LSTM_BC][H]
    float* gs = hs + (size_t)LSTM_BC * H;   // [R][LSTM_BC]
    float* cs = gs + R * LSTM_BC;           // [U][B] cell state

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int unit0 = blockIdx.x * U;
    const unsigned ncta = gridDim.x;

    for (int idx = tid; idx < R * (H / 4); idx += 256) {
        int r = idx / (H / 4), c4 = idx - r * (H / 4);
        int gate = r / U, u = r - gate * U;
        reinterpret_cast<float4*>(wsm)[idx] =
            reinterpret_cast<const float4*>(p.whh + ((size_t)gate * H + unit0 + u) * H)[c4];
    }
    for (int idx = tid; idx < U * p.B; idx += 256) cs[idx] = 0.f;
    __syncthreads();

    for (int t = 0; t < p.T; ++t) {
        const float* hprev = p.hbuf + (size_t)(t & 1) * p.B * H;
        float* hnext = p.hbuf + (size_t)((t + 1) & 1) * p.B * H;
        for (int b0 = 0; b0 < p.B; b0 += LSTM_BC) {
            const int nb = min(LSTM_BC, p.B - b0);
            // gate inputs for this CTA's (unit, batch) pairs: issued early, consumed after the matvec
            float gxr[4] = {0.f, 0.f, 0.f, 0.f};
            const int pu = tid / LSTM_BC, pb = tid % LSTM_BC;
            const bool pw = (tid < U * LSTM_BC) && (pb < nb);
            if (pw) {
#pragma unroll
                for (int g = 0; g < 4; ++g)
                    gxr[g] = __ldg(p.gx + ((size_t)(b0 + pb) * 4 * H + (size_t)g * H + unit0 + pu) * p.T + t);
            }
            if (t > 0) {
                for (int idx = tid; idx < LSTM_BC * (H / 4); idx += 256) {
                    int bb = idx / (H / 4), c4 = idx - bb * (H / 4);
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (bb < nb) v = __ldcg(reinterpret_cast<const float4*>(hprev + (size_t)(b0 + bb) * H) + c4);
                    reinterpret_cast<float4*>(hs)[idx] = v;
                }
                __syncthreads();
                for (int r0 = warp * 4; r0 < R; r0 += 32) {
                    float acc[4 * LSTM_BC];
#pragma unroll
                    for (int i = 0; i < 4 * LSTM_BC; ++i) acc[i] = 0.f;
                    for (int kk = lane * 4; kk < H; kk += 128) {
                        float4 w4[4];
#pragma unroll
                        for (int r = 0; r < 4; ++r) w4[r] = *reinterpret_cast<const float4*>(wsm + (size_t)(r0 + r) * H + kk);
#pragma unroll
                        for (int bb = 0; bb < LSTM_BC; ++bb) {
                            const float4 h4 = *reinterpret_cast<const float4*>(hs + (size_t)bb * H + kk);
#pragma unroll
                            for (int r = 0; r < 4; ++r) {
                                float a = acc[r * LSTM_BC + bb];
                                a = fmaf(w4[r].x, h4.x, a);
                                a = fmaf(w4[r].y, h4.y, a);
                                a = fmaf(w4[r].z, h4.z, a);
                                a = fmaf(w4[r].w, h4.w, a);
                                acc[r * LSTM_BC + bb] = a;
                            }
                        }
                    }
                    // transpose-reduce 32 values at a time: afterwards lane l holds the warp-wide sum of acc[half*32 + l]
#pragma unroll
                    for (int half = 0; half < (4 * LSTM_BC) / 32; ++half) {
#pragma unroll
                        for (int off = 16, n = 16; off >= 1; off >>= 1, n >>= 1) {
                            const bool upper = (lane & off) != 0;
#pragma unroll
                            for (int i = 0; i < n; ++i) {
                                float send = upper ? acc[half * 32 + i] : acc[half * 32 + i + n];
                                float keep = upper ? acc[half * 32 + i + n] : acc[half * 32 + i];
                                acc[half * 32 + i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                            }
                        }
                        const int vi = half * 32 + lane;   // value index = r * LSTM_BC + bb
                        gs[(r0 + vi / LSTM_BC) * LSTM_BC + (vi % LSTM_BC)] = acc[half * 32];
                    }
                }
                __syncthreads();
            }
            if (pw) {
                float gi = gxr[0], gf = gxr[1], gg = gxr[2], go = gxr[3];
                if (t > 0) {
                    gi += gs[(0 * U + pu) * LSTM_BC + pb];
                    gf += gs[(1 * U + pu) * LSTM_BC + pb];
                    gg += gs[(2 * U + pu) * LSTM_BC + pb];
                    go += gs[(3 * U + pu) * LSTM_BC + pb];
                }
                float c = cs[pu * p.B + b0 + pb];
                c = sigmoidf_(gf) * c + sigmoidf_(gi) * tanhf(gg);
                float h = sigmoidf_(go) * tanhf(c);
                cs[pu * p.B + b0 + pb] = c;
                __stcg(hnext + (size_t)(b0 + pb) * H + unit0 + pu, h);
                size_t yo = ((size_t)(b0 + pb) * H + unit0 + pu) * p.T + t;
                p.y[yo] = p.skip ? h + p.skip[yo] : h;
            }
            __syncthreads();  // gs / hs reused by the next batch chunk
        }
        // grid barrier: everyone has published h_t before anyone reads it
        if (tid == 0) {
            __threadfence();
            atomicAdd(p.bar, 1u);
            const unsigned target = ncta * (unsigned)(t + 1);
            while (ld_acquire_u32(p.bar) < target) { }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// Recurrent LSTM step on the tensor pipe (hidden % 64 == 0, batch <= 32): 3xTF32 mma.sync.m16n8k8, fp32 accumulate.
//   gates[32 rows = 4 gates x 8 units of this CTA][32 items] = W_hh slice [32][H] . h_{t-1} [H][32]
// * CTA = 8 units (H / 8 CTAs, co-resident: cooperative launch), 8 warps; warp w multiplies the K range [w H/8, (w+1) H/8) for all
//   32 rows x 32 items (2 m16 x 4 n8 tiles, 32 accumulator registers); the 8 partial tiles are summed in shared memory in warp order.
// * W_hh slice resident in shared memory for the whole sequence (row pitch H + 4 floats: conflict-free A fragments), split into tf32
//   hi / lo terms on the way into the MMA.
// * h lives in global memory in the B-FRAGMENT order hF[k / 8][k % 8][item % 8][item / 8]: lane (g, c) fetches its four n-tiles of
//   k-row c (resp. c + 4) with one 16-byte load, a warp instruction reads 4 x 128 contiguous bytes, every byte fetched is used
//   (128 KB per CTA and step, the minimum for "every CTA needs all of h"), and nothing is staged through shared memory.
// * thread (unit u = tid / 32, item b = tid % 32) owns one cell: its c_t stays in a register for the whole sequence, it adds the
//   input half of the gates (requested one step ahead), applies the nonlinearities and writes h_t (fragment order) and y.
// * one grid barrier per step (release arrive / acquire poll), h double-buffered.
// The fp32 FMA kernel above makes two 16-item passes per step at H = 1024 (each: stage 64 KB of h, 2 048 FFMA per thread,
// transposing reduction); this one reads h once and does the arithmetic on the tensor pipe.
// ------------------------------------------------------------------------------------------------
constexpr int LTC_U = 8, LTC_ROWS = 4 * LTC_U, LTC_B = 32, LTC_NW = 8, LTC_PB = 4;   // 8 warps; B fragments of LTC_PB k-steps requested together
__global__ void __launch_bounds__(LTC_NW * 32, 1) lstm_tc_kernel(LstmParams p) {
    extern __shared__ float smem[];
    const int H = p.H, WP = H + 4;
    float* wsm = smem;                           // [32][WP]
    float* red = wsm + (size_t)LTC_ROWS * WP;    // [8 warps][32 rows][33]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
    const int unit0 = blockIdx.x * LTC_U;
    const unsigned ncta = gridDim.x;

    for (int idx = tid; idx < LTC_ROWS * (H / 4); idx += LTC_NW * 32) {
        const int r = idx / (H / 4), c4 = idx - r * (H / 4), gate = r / LTC_U, u = r - gate * LTC_U;
        const float4 w = __ldg(reinterpret_cast<const float4*>(p.whh + ((size_t)gate * H + unit0 + u) * H) + c4);
        *reinterpret_cast<float4*>(wsm + (size_t)r * WP + 4 * c4) = w;
    }
    __syncthreads();

    const int cu = (tid >> 5) & (LTC_U - 1), cb = tid & 31;   // threads 0..255 own one cell each: unit unit0 + cu, item cb
    const bool cell_live = tid < LTC_U * 32 && cb < p.B;
    const int kunit = unit0 + cu;
    const size_t hf_cell = ((size_t)kunit * 8 + (cb & 7)) * 4 + (cb >> 3);   // hF float index of (k = kunit, item cb)
    const size_t hf_size = (size_t)H * LTC_B;
    const size_t gx_cell = ((size_t)cb * 4 * H + kunit) * p.T;               // + gate * H * T + t
    const size_t y_cell = ((size_t)cb * H + kunit) * p.T;
    float cstate = 0.f;
    const int ksteps = H / (8 * LTC_NW);         // k-steps of 8 per warp
    const int kb0 = warp * ksteps;               // first k-block (of 8) of this warp

    float gxr[4] = {0.f, 0.f, 0.f, 0.f};
    if (cell_live) {
#pragma unroll
        for (int gt = 0; gt < 4; ++gt) gxr[gt] = __ldg(p.gx + gx_cell + (size_t)gt * H * p.T);
    }
    for (int t = 0; t < p.T; ++t) {
        const float* hprev = p.hbuf + (size_t)(t & 1) * hf_size;
        float* hnext = p.hbuf + (size_t)((t + 1) & 1) * hf_size;
        float gi = gxr[0], gf = gxr[1], gg = gxr[2], go = gxr[3];
        if (cell_live && t + 1 < p.T) {          // next step's input half: in flight during this step's MMAs
#pragma unroll
            for (int gt = 0; gt < 4; ++gt) gxr[gt] = __ldg(p.gx + gx_cell + (size_t)gt * H * p.T + t + 1);
        }
        if (t > 0) {
            float acc[2][4][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
            const float4* hf4 = reinterpret_cast<const float4*>(hprev);
            // B fragments are requested LTC_PB k-steps at a time (8 warps x 4 k-steps): all k-steps up front needs 255 registers,
            // 16 warps spill, and two alternating item halves split W_hh twice per step; each of those was measured slower on the
            // previous GPU generation (not re-measured on the H100).
#pragma unroll 1
            for (int s0 = 0; s0 < ksteps; s0 += LTC_PB) {
                float4 b0[LTC_PB], b1[LTC_PB];
#pragma unroll
                for (int s = 0; s < LTC_PB; ++s) {
                    if (s0 + s < ksteps) {       // warp-uniform
                        const size_t kb = (size_t)(kb0 + s0 + s);
                        b0[s] = __ldcg(hf4 + (kb * 8 + c) * 8 + g);
                        b1[s] = __ldcg(hf4 + (kb * 8 + c + 4) * 8 + g);
                    }
                }
#pragma unroll
                for (int s = 0; s < LTC_PB; ++s) {
                    if (s0 + s >= ksteps) break;
                    const int k = (kb0 + s0 + s) * 8;
                    uint32_t ah[2][4], al[2][4];
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) {
                        const float* wr = wsm + (size_t)(mt * 16 + g) * WP + k + c;
                        rb_split(wr[0], ah[mt][0], al[mt][0]);
                        rb_split(wr[8 * WP], ah[mt][1], al[mt][1]);
                        rb_split(wr[4], ah[mt][2], al[mt][2]);
                        rb_split(wr[8 * WP + 4], ah[mt][3], al[mt][3]);
                    }
                    const float bx0[4] = {b0[s].x, b0[s].y, b0[s].z, b0[s].w}, bx1[4] = {b1[s].x, b1[s].y, b1[s].z, b1[s].w};
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                        uint32_t bh0, bl0, bh1, bl1;
                        rb_split(bx0[nt], bh0, bl0);
                        rb_split(bx1[nt], bh1, bl1);
#pragma unroll
                        for (int mt = 0; mt < 2; ++mt) {
                            mma_tf32(acc[mt][nt], al[mt], bh0, bh1);
                            mma_tf32(acc[mt][nt], ah[mt], bl0, bl1);
                            mma_tf32(acc[mt][nt], ah[mt], bh0, bh1);
                        }
                    }
                }
            }
            float* rw = red + (size_t)warp * LTC_ROWS * 33;
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    float* r0 = rw + (mt * 16 + g) * 33 + nt * 8 + 2 * c;
                    r0[0] = acc[mt][nt][0];
                    r0[1] = acc[mt][nt][1];
                    r0[8 * 33] = acc[mt][nt][2];
                    r0[8 * 33 + 1] = acc[mt][nt][3];
                }
            __syncthreads();
#pragma unroll
            for (int w = 0; w < LTC_NW; ++w) {   // warp order: fixed summation order
                const float* rr = red + (size_t)w * LTC_ROWS * 33 + cb;
                gi += rr[(0 * LTC_U + cu) * 33];
                gf += rr[(1 * LTC_U + cu) * 33];
                gg += rr[(2 * LTC_U + cu) * 33];
                go += rr[(3 * LTC_U + cu) * 33];
            }
        }
        if (cell_live) {
            cstate = sigmoidf_(gf) * cstate + sigmoidf_(gi) * tanhf(gg);
            const float h = sigmoidf_(go) * tanhf(cstate);
            __stcg(hnext + hf_cell, h);
            p.y[y_cell + t] = p.skip ? h + p.skip[y_cell + t] : h;
        }
        // grid barrier: everyone has published h_t (and is done with the partial-sum buffer) before anyone reads it
        __syncthreads();
        if (tid == 0) {   // release reduction without a return value + acquire polling (csrc/gridbar.cuh): no membar.gl, no atomic round trip
            gridbar_arrive(p.bar);
            gridbar_wait(p.bar, ncta * (unsigned)(t + 1));
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// Recurrent LSTM step with BOTH operands pre-split into two fp16 terms (hidden % 128 == 0, batch <= 32): the default since the end of
// round 2.  x = hi + lo * 2^-11 with hi = fp16(x), lo = fp16((x - hi) * 2^11): 22 mantissa bits, the precision class of the 3xTF32
// split (tf32 carries 11), and |W_hh| <~ 1, |h| < 1 sit inside fp16's range (the scaled low terms too).  Then
//     W h = (hi_w hi_h) + 2^-11 (hi_w lo_h + lo_w hi_h)            [lo lo dropped: 2^-22]
// is THREE mma.sync.m16n8k16.f16 per 16 reduction elements (the tf32 kernel: six m16n8k8), and -- the actual point -- nothing is
// converted inside the step any more:
//   * W_hh's slice is split ONCE, at kernel start, straight into the A-fragment order of its consumer warp:
//     wfrag[warp][k16 step][m tile][hi | lo][lane][4 x half2], 4 bytes per element like the fp32 copy (128 KB at H = 1024), one
//     conflict-free LDS.128 per term and m tile;
//   * h_t is split by the ONE thread that produces it and stored in the B-fragment order of m16n8k16,
//     hF[k / 16][hi | lo][b0 | b1][(k % 8) / 2][item % 8][item / 8] (half2 = the two k of a register), so a lane fetches the four
//     n-tiles of a fragment register with one 16-byte load (4 loads per k16 step, every byte used).
// lstm_tc_kernel spent ~900 instructions per 4 k8 steps for 96 HMMA (ncu: 30 % of the stall samples on HMMA, 29 % fixed-latency waits
// of the conversion chains); here a k16 step is 4 LDG.128 + 4 LDS.128 + 24 HMMA.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_f16(float (&c)[4], const uint4& a, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void split_h2(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn((v - __half2float(hi)) * 2048.f);
}
constexpr int LH2_PB = 4;   // k16 steps of B fragments requested together (all 8 at once needs 254 registers and was slower)
__global__ void __launch_bounds__(LTC_NW * 32, 1) lstm_h2_kernel(LstmParams p) {
    extern __shared__ float smem[];
    const int H = p.H;
    uint4* wfrag = reinterpret_cast<uint4*>(smem);                 // [warp][k16 step][m tile][hi | lo][lane]
    float* red = smem + (size_t)LTC_ROWS * H;                      // [8 warps][32 rows][33]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
    const int unit0 = blockIdx.x * LTC_U;
    const unsigned ncta = gridDim.x;
    const int ksteps = H / (16 * LTC_NW);        // k16 steps per warp
    const int kb0 = warp * ksteps;               // first k16 block of this warp

    // ---- W_hh slice -> fp16 hi / lo A fragments (once).  Fragment registers of m16n8k16: a0 = (row g, k 2c..2c+1), a1 = (g + 8, 2c..),
    //      a2 = (g, 2c + 8..), a3 = (g + 8, 2c + 8..); tile row r = gate * 8 + unit  ->  W_hh row gate * H + unit0 + unit.
    for (int s = 0; s < ksteps; ++s)
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            __half2 hi[4], lo[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int r = mt * 16 + g + (j & 1) * 8, gate = r / LTC_U, u = r - gate * LTC_U;
                const int k = (kb0 + s) * 16 + 2 * c + (j >> 1) * 8;
                const float2 w = __ldg(reinterpret_cast<const float2*>(p.whh + ((size_t)gate * H + unit0 + u) * H + k));
                __half h0, l0, h1, l1;
                split_h2(w.x, h0, l0);
                split_h2(w.y, h1, l1);
                hi[j] = __halves2half2(h0, h1);
                lo[j] = __halves2half2(l0, l1);
            }
            uint4* dst = wfrag + ((size_t)((warp * ksteps + s) * 2 + mt) * 2) * 32 + lane;
            dst[0] = make_uint4(*reinterpret_cast<uint32_t*>(&hi[0]), *reinterpret_cast<uint32_t*>(&hi[1]),
                                *reinterpret_cast<uint32_t*>(&hi[2]), *reinterpret_cast<uint32_t*>(&hi[3]));
            dst[32] = make_uint4(*reinterpret_cast<uint32_t*>(&lo[0]), *reinterpret_cast<uint32_t*>(&lo[1]),
                                 *reinterpret_cast<uint32_t*>(&lo[2]), *reinterpret_cast<uint32_t*>(&lo[3]));
        }
    __syncthreads();

    const int cu = (tid >> 5) & (LTC_U - 1), cb = tid & 31;   // threads 0..255 own one cell each: unit unit0 + cu, item cb
    const bool cell_live = tid < LTC_U * 32 && cb < p.B;
    const int kunit = unit0 + cu;
    // hF half index of (k = kunit, item cb), hi term; the lo term sits 2 * 4 * 8 * 4 * 2 = 512 halves further
    const size_t hf_cell = ((((size_t)(kunit >> 4) * 2 * 2 + ((kunit & 15) >> 3)) * 4 + ((kunit & 7) >> 1)) * 8 + (cb & 7)) * 8 +
                           (size_t)(cb >> 3) * 2 + (kunit & 1);
    const size_t hf_size = (size_t)H * LTC_B * 2;             // halves per buffer
    const size_t gx_cell = ((size_t)cb * 4 * H + kunit) * p.T;
    const size_t y_cell = ((size_t)cb * H + kunit) * p.T;
    float cstate = 0.f;
    __half* hbuf = reinterpret_cast<__half*>(p.hbuf);

    float gxr[4] = {0.f, 0.f, 0.f, 0.f};
    if (cell_live) {
#pragma unroll
        for (int gt = 0; gt < 4; ++gt) gxr[gt] = __ldg(p.gx + gx_cell + (size_t)gt * H * p.T);
    }
    for (int t = 0; t < p.T; ++t) {
        const __half* hprev = hbuf + (size_t)(t & 1) * hf_size;
        __half* hnext = hbuf + (size_t)((t + 1) & 1) * hf_size;
        float gi = gxr[0], gf = gxr[1], gg = gxr[2], go = gxr[3];
        if (cell_live && t + 1 < p.T) {
#pragma unroll
            for (int gt = 0; gt < 4; ++gt) gxr[gt] = __ldg(p.gx + gx_cell + (size_t)gt * H * p.T + t + 1);
        }
        if (t > 0) {
            float acc0[2][4][4], acc1[2][4][4];   // hi.hi | hi.lo + lo.hi (scaled by 2^11)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    acc0[i][j][0] = acc0[i][j][1] = acc0[i][j][2] = acc0[i][j][3] = 0.f;
                    acc1[i][j][0] = acc1[i][j][1] = acc1[i][j][2] = acc1[i][j][3] = 0.f;
                }
            const uint4* hf4 = reinterpret_cast<const uint4*>(hprev);   // [k16][hi|lo][b][c][g] of uint4 (4 n tiles)
#pragma unroll 1
            for (int s0 = 0; s0 < ksteps; s0 += LH2_PB) {
                uint4 bf[LH2_PB][4];             // [step][hi b0, hi b1, lo b0, lo b1]
#pragma unroll
                for (int s = 0; s < LH2_PB; ++s) {
                    if (s0 + s < ksteps) {       // warp-uniform
                        const uint4* q = hf4 + (size_t)(kb0 + s0 + s) * 128 + c * 8 + g;
#pragma unroll
                        for (int j = 0; j < 4; ++j) bf[s][j] = __ldcg(q + j * 32);
                    }
                }
#pragma unroll
                for (int s = 0; s < LH2_PB; ++s) {
                    if (s0 + s >= ksteps) break;
                    const uint4* wf = wfrag + ((size_t)(warp * ksteps + s0 + s) * 2 * 2) * 32 + lane;
                    const uint4 ah0 = wf[0], al0 = wf[32], ah1 = wf[64], al1 = wf[96];
                    const uint32_t hb0[4] = {bf[s][0].x, bf[s][0].y, bf[s][0].z, bf[s][0].w};
                    const uint32_t hb1[4] = {bf[s][1].x, bf[s][1].y, bf[s][1].z, bf[s][1].w};
                    const uint32_t lb0[4] = {bf[s][2].x, bf[s][2].y, bf[s][2].z, bf[s][2].w};
                    const uint32_t lb1[4] = {bf[s][3].x, bf[s][3].y, bf[s][3].z, bf[s][3].w};
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                        mma_f16(acc0[0][nt], ah0, hb0[nt], hb1[nt]);
                        mma_f16(acc0[1][nt], ah1, hb0[nt], hb1[nt]);
                        mma_f16(acc1[0][nt], ah0, lb0[nt], lb1[nt]);
                        mma_f16(acc1[1][nt], ah1, lb0[nt], lb1[nt]);
                        mma_f16(acc1[0][nt], al0, hb0[nt], hb1[nt]);
                        mma_f16(acc1[1][nt], al1, hb0[nt], hb1[nt]);
                    }
                }
            }
            float* rw = red + (size_t)warp * LTC_ROWS * 33;
            constexpr float LO = 1.f / 2048.f;
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    float* r0 = rw + (mt * 16 + g) * 33 + nt * 8 + 2 * c;
                    r0[0] = fmaf(acc1[mt][nt][0], LO, acc0[mt][nt][0]);
                    r0[1] = fmaf(acc1[mt][nt][1], LO, acc0[mt][nt][1]);
                    r0[8 * 33] = fmaf(acc1[mt][nt][2], LO, acc0[mt][nt][2]);
                    r0[8 * 33 + 1] = fmaf(acc1[mt][nt][3], LO, acc0[mt][nt][3]);
                }
            __syncthreads();
#pragma unroll
            for (int w = 0; w < LTC_NW; ++w) {   // warp order: fixed summation order
                const float* rr = red + (size_t)w * LTC_ROWS * 33 + cb;
                gi += rr[(0 * LTC_U + cu) * 33];
                gf += rr[(1 * LTC_U + cu) * 33];
                gg += rr[(2 * LTC_U + cu) * 33];
                go += rr[(3 * LTC_U + cu) * 33];
            }
        }
        if (cell_live) {
            cstate = sigmoidf_(gf) * cstate + sigmoidf_(gi) * tanhf(gg);
            const float h = sigmoidf_(go) * tanhf(cstate);
            __half hh, hl;
            split_h2(h, hh, hl);
            hnext[hf_cell] = hh;                 // plain stores: published by the release arrive below
            hnext[hf_cell + 512] = hl;
            p.y[y_cell + t] = p.skip ? h + p.skip[y_cell + t] : h;
        }
        __syncthreads();
        if (tid == 0) {
            gridbar_arrive(p.bar);
            gridbar_wait(p.bar, ncta * (unsigned)(t + 1));
        }
        __syncthreads();
    }
}

extern "C" int64_t acb_lstm_state_bytes(int batch, int hidden) {
    const int64_t b = batch > LTC_B ? batch : LTC_B;   // the tensor-core kernel keeps h for 32 item slots
    return ((int64_t)2 * b * hidden + 64) * (int64_t)sizeof(float);
}

extern "C" int acb_lstm_recurrent(const float* gates_x, const float* w_hh, const float* skip, float* y,
                                  float* state_ws, int batch, int hidden, int t_len, void* stream) {
    ACB_REQUIRE(gates_x && w_hh && y && state_ws, "acb_lstm_recurrent: null pointer");
    ACB_REQUIRE(batch > 0 && hidden > 0 && t_len > 0, "acb_lstm_recurrent: empty shape");
    ACB_REQUIRE(hidden % 4 == 0, "acb_lstm_recurrent: hidden must be a multiple of 4");
    cudaStream_t s = (cudaStream_t)stream;
    {   // tensor-core kernel: hidden a multiple of 64, up to 32 items, H / 8 co-resident CTAs; ACB_LSTM_TC=0 keeps the fp32 FMA kernel
        const char* e = getenv("ACB_LSTM_TC");
        const size_t smem_tc = ((size_t)LTC_ROWS * (hidden + 4) + (size_t)LTC_NW * LTC_ROWS * 33) * sizeof(float);
        if (!(e && e[0] == '0') && hidden % (8 * LTC_NW) == 0 && batch <= LTC_B && smem_tc <= 227 * 1024) {
            const int ncta = hidden / LTC_U;
            ACB_CHECK_CUDA(cudaFuncSetAttribute(lstm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tc));
            int dev = 0, sms = 0, per_sm = 0;
            ACB_CHECK_CUDA(cudaGetDevice(&dev));
            ACB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
            ACB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lstm_tc_kernel, LTC_NW * 32, smem_tc));
            if (per_sm * sms >= ncta) {
                const size_t hfloats = (size_t)2 * LTC_B * hidden;
                ACB_CHECK_CUDA(cudaMemsetAsync(state_ws, 0, (hfloats + 64) * sizeof(float), s));
                LstmParams p{gates_x, w_hh, skip, y, state_ws, (unsigned*)(state_ws + hfloats), batch, hidden, t_len, LTC_U};
                void* args[] = {&p};
                // hidden % 128 == 0: both operands pre-split into fp16 terms (lstm_h2_kernel); ACB_LSTM_TC=3 keeps the 3xTF32 kernel (A/B)
                const bool h2 = hidden % (16 * LTC_NW) == 0 && !(e && e[0] == '3');
                if (h2) ACB_CHECK_CUDA(cudaFuncSetAttribute(lstm_h2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tc));
                ACB_CHECK_CUDA(cudaLaunchCooperativeKernel(h2 ? (void*)lstm_h2_kernel : (void*)lstm_tc_kernel, dim3(ncta), dim3(LTC_NW * 32),
                                                           args, smem_tc, s));
                return ACB_OK;
            }
        }
    }
    int U = hidden >= 128 ? hidden / 128 : 1;
    ACB_REQUIRE(hidden % U == 0, "acb_lstm_recurrent: hidden %d not divisible by %d units per CTA", hidden, U);
    int ncta = hidden / U;
    size_t smem = ((size_t)4 * U * hidden + (size_t)LSTM_BC * hidden + (size_t)4 * U * LSTM_BC + (size_t)U * batch) *
                  sizeof(float);
    ACB_REQUIRE(smem <= 227 * 1024, "acb_lstm_recurrent: hidden=%d batch=%d needs %zu B smem per CTA", hidden, batch, smem);
    ACB_REQUIRE(U * LSTM_BC <= 256, "acb_lstm_recurrent: too many units per CTA");
    ACB_CHECK_CUDA(cudaFuncSetAttribute(lstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0, sms = 0, per_sm = 0;
    ACB_CHECK_CUDA(cudaGetDevice(&dev));
    ACB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    ACB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lstm_kernel, 256, smem));
    ACB_REQUIRE(per_sm * sms >= ncta, "acb_lstm_recurrent: %d CTAs cannot be co-resident (%d SMs x %d)", ncta, sms, per_sm);
    size_t hbytes = (size_t)2 * batch * hidden * sizeof(float);
    ACB_CHECK_CUDA(cudaMemsetAsync(state_ws, 0, hbytes + 64 * sizeof(float), s));
    LstmParams p{gates_x, w_hh, skip, y, state_ws, (unsigned*)(state_ws + (size_t)2 * batch * hidden), batch, hidden,
                 t_len, U};
    void* args[] = {&p};
    ACB_CHECK_CUDA(cudaLaunchCooperativeKernel((void*)lstm_kernel, dim3(ncta), dim3(256), args, smem, s));
    return ACB_OK;
}

// ------------------------------------------------------------------------------------------------
// RVQ encode: CTA = 32 frames; residuals live in smem for all n_q rounds; the codebook streams through
// smem in tiles of 64 codes (from L2: 4 x 1 MB codebooks stay resident there).  Thread (warp w, lane f)
// scores frame f against 8 codes of every tile.
// ------------------------------------------------------------------------------------------------
constexpr int RVQ_F = 32, RVQ_TILE = 64;

__global__ void __launch_bounds__(256) rvq_encode_kernel(const float* __restrict__ z, const float* __restrict__ cb,
                                                         const float* __restrict__ cbn, int64_t* __restrict__ codes,
                                                         int B, int D, int T, int n_q, int bins) {
    extern __shared__ float smem[];
    float* rs = smem;                      // [D][32] residual, frame fastest
    float* cs = rs + D * RVQ_F;            // [RVQ_TILE][D+1]
    float* bs = cs + RVQ_TILE * (D + 1);   // [8][32] best score per warp
    int* bi = (int*)(bs + 8 * RVQ_F);      // [8][32] best index per warp
    int* sel = bi + 8 * RVQ_F;             // [32] chosen code per frame

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long n0 = (long long)blockIdx.x * RVQ_F;
    const long long N = (long long)B * T;
    const long long n = n0 + lane;
    const bool live = n < N;
    const int fb = live ? (int)(n / T) : 0, ft = live ? (int)(n % T) : 0;

    for (int d = warp; d < D; d += 8) rs[d * RVQ_F + lane] = live ? z[((size_t)fb * D + d) * T + ft] : 0.f;
    __syncthreads();

    for (int q = 0; q < n_q; ++q) {
        const float* cbq = cb + (size_t)q * bins * D;
        float xx = 0.f;
        for (int d = 0; d < D; ++d) { float r = rs[d * RVQ_F + lane]; xx = fmaf(r, r, xx); }
        float best = -INFINITY;
        int besti = 0;
        for (int c0 = 0; c0 < bins; c0 += RVQ_TILE) {
            __syncthreads();
            for (int idx = tid; idx < RVQ_TILE * D; idx += 256) {
                int c = idx / D, d = idx - c * D;
                cs[c * (D + 1) + d] = (c0 + c < bins) ? cbq[(size_t)(c0 + c) * D + d] : 0.f;
            }
            __syncthreads();
            float dot[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) dot[i] = 0.f;
            const float* cw = cs + (warp * 8) * (D + 1);
            for (int d = 0; d < D; ++d) {
                float r = rs[d * RVQ_F + lane];
#pragma unroll
                for (int i = 0; i < 8; ++i) dot[i] = fmaf(r, cw[i * (D + 1) + d], dot[i]);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                int c = c0 + warp * 8 + i;
                if (c < bins) {
                    // same association as core_vq.py:166-170: -((|x|^2 - 2 x.e) + |e|^2)
                    float sc = -((xx - 2.f * dot[i]) + cbn[(size_t)q * bins + c]);
                    if (sc > best) { best = sc; besti = c; }
                }
            }
        }
        bs[warp * RVQ_F + lane] = best;
        bi[warp * RVQ_F + lane] = besti;
        __syncthreads();
        if (warp == 0) {
            float m = bs[lane];
            int mi = bi[lane];
            for (int w = 1; w < 8; ++w) {
                float v = bs[w * RVQ_F + lane];
                int vi = bi[w * RVQ_F + lane];
                if (v > m || (v == m && vi < mi)) { m = v; mi = vi; }  // first max wins (torch.max)
            }
            sel[lane] = mi;
            if (live) codes[((size_t)fb * n_q + q) * T + ft] = mi;
        }
        __syncthreads();
        const int mine = sel[lane];
        for (int d = warp; d < D; d += 8) rs[d * RVQ_F + lane] -= cbq[(size_t)mine * D + d];
        __syncthreads();
    }
}

extern "C" int acb_rvq_encode(const float* latent, const float* codebooks, const float* cb_sqnorm, int64_t* codes,
                              int batch, int dim, int t_len, int n_q, int bins, void* stream) {
    ACB_REQUIRE(latent && codebooks && cb_sqnorm && codes, "acb_rvq_encode: null pointer");
    ACB_REQUIRE(batch > 0 && t_len > 0 && n_q > 0 && bins > 0, "acb_rvq_encode: empty shape");
    ACB_REQUIRE(dim > 0 && dim <= 512, "acb_rvq_encode: dim %d out of range (<=512)", dim);
    size_t smem = ((size_t)dim * RVQ_F + (size_t)RVQ_TILE * (dim + 1) + 8 * RVQ_F) * sizeof(float) +
                  (8 * RVQ_F + RVQ_F) * sizeof(int);
    if (smem > 48 * 1024)
        ACB_CHECK_CUDA(cudaFuncSetAttribute(rvq_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    long long N = (long long)batch * t_len;
    rvq_encode_kernel<<<(unsigned)((N + RVQ_F - 1) / RVQ_F), 256, smem, (cudaStream_t)stream>>>(
        latent, codebooks, cb_sqnorm, codes, batch, dim, t_len, n_q, bins);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

// RVQ decode: latent[b][d][t] = sum_k E_k[codes[b][k][t]][d]; 32 frames per CTA, transposed through smem so
// both the codebook row reads and the [B][D][T] writes are coalesced.
__global__ void __launch_bounds__(256) rvq_decode_kernel(const int64_t* __restrict__ codes, const float* __restrict__ cb,
                                                         float* __restrict__ out, int B, int D, int T, int n_q,
                                                         int bins) {
    extern __shared__ float smem[];  // [32][D+1]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long n0 = (long long)blockIdx.x * 32, N = (long long)B * T;
    for (int f = warp; f < 32; f += 8) {
        long long n = n0 + f;
        if (n >= N) continue;
        int b = (int)(n / T), t = (int)(n % T);
        for (int d = lane; d < D; d += 32) {
            float acc = 0.f;
            for (int q = 0; q < n_q; ++q) {
                long long c = codes[((size_t)b * n_q + q) * T + t];
                c = c < 0 ? 0 : (c >= bins ? bins - 1 : c);
                acc += cb[((size_t)q * bins + c) * D + d];
            }
            smem[f * (D + 1) + d] = acc;
        }
    }
    __syncthreads();
    long long n = n0 + lane;
    if (n < N) {
        int b = (int)(n / T), t = (int)(n % T);
        for (int d = warp; d < D; d += 8) out[((size_t)b * D + d) * T + t] = smem[lane * (D + 1) + d];
    }
}

extern "C" int acb_rvq_decode(const int64_t* codes, const float* codebooks, float* latent, int batch, int dim, int t_len,
                              int n_q, int bins, void* stream) {
    ACB_REQUIRE(codes && codebooks && latent, "acb_rvq_decode: null pointer");
    ACB_REQUIRE(batch > 0 && dim > 0 && t_len > 0 && n_q > 0 && bins > 0, "acb_rvq_decode: empty shape");
    size_t smem = (size_t)32 * (dim + 1) * sizeof(float);
    ACB_REQUIRE(smem <= 48 * 1024, "acb_rvq_decode: dim %d too large", dim);
    long long N = (long long)batch * t_len;
    rvq_decode_kernel<<<(unsigned)((N + 31) / 32), 256, smem, (cudaStream_t)stream>>>(codes, codebooks, latent, batch, dim,
                                                                                     t_len, n_q, bins);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

// ------------------------------------------------------------------------------------------------
// GroupNorm(1, C) of a SEANet layer output (norm='time_group_norm', modules/conv.py:33-42; NormConv1d /
// NormConvTranspose1d apply it after the convolution and, for the transposed conv, before the trim).
// Statistics of item b over its C*T elements in two deterministic passes: GN_PART blocks per item
// (a count that depends on C*T only, never on the batch) each reduce a fixed contiguous slice in a
// fixed order into fp64 sums of x - x[b][0][0] (shifted by the item's first sample, so a large mean
// does not cancel the variance), then one warp per item combines the partials in a fixed order.
// ------------------------------------------------------------------------------------------------
constexpr int GN_THREADS = 256;
constexpr int GN_MAX_PARTS = 256;

static int gn_parts(long long n) {
    long long p = (n + 16383) / 16384;   // >= 16 K elements per block
    return (int)(p < 1 ? 1 : (p > GN_MAX_PARTS ? GN_MAX_PARTS : p));
}

__global__ void __launch_bounds__(GN_THREADS) groupnorm_partial_kernel(const float* __restrict__ x, double2* __restrict__ part,
                                                                        long long n, int parts) {
    __shared__ double2 red[GN_THREADS / 32];
    const int p = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const float* xb = x + (size_t)b * n;
    const long long chunk = (n + parts - 1) / parts;
    const long long lo = (long long)p * chunk, hi = min(n, lo + chunk);
    const double shift = (double)__ldg(xb);
    double s1 = 0.0, s2 = 0.0;
    long long i = lo + tid;
    for (; i + 3 * GN_THREADS < hi; i += 4 * GN_THREADS) {   // four independent loads in flight per thread
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = __ldg(xb + i + u * GN_THREADS);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const double d = (double)v[u] - shift;
            s1 += d;
            s2 = fma(d, d, s2);
        }
    }
    for (; i < hi; i += GN_THREADS) {
        const double d = (double)__ldg(xb + i) - shift;
        s1 += d;
        s2 = fma(d, d, s2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if ((tid & 31) == 0) red[tid >> 5] = make_double2(s1, s2);
    __syncthreads();
    if (tid == 0) {
        double a = 0.0, q = 0.0;
        for (int w = 0; w < GN_THREADS / 32; ++w) { a += red[w].x; q += red[w].y; }
        part[(size_t)b * parts + p] = make_double2(a, q);
    }
}

__global__ void groupnorm_finalize_kernel(const float* __restrict__ x, const double2* __restrict__ part, double2* __restrict__ stats,
                                          long long n, int parts, int batch, float eps) {
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= batch) return;
    double s1 = 0.0, s2 = 0.0;
    for (int p = lane; p < parts; p += 32) {
        const double2 v = part[(size_t)b * parts + p];
        s1 += v.x;
        s2 += v.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) {
        const double m = s1 / (double)n;
        const double var = fmax(s2 / (double)n - m * m, 0.0);   // biased variance, as nn.GroupNorm
        stats[b] = make_double2((double)x[(size_t)b * n] + m, 1.0 / sqrt(var + (double)eps));
    }
}

extern "C" int64_t acb_groupnorm_workspace_bytes(int batch, int channels, int t_len) {
    if (batch <= 0 || channels <= 0 || t_len <= 0) return 0;
    return (int64_t)batch * gn_parts((long long)channels * t_len) * (int64_t)sizeof(double2);
}

extern "C" int acb_groupnorm_stats(const float* x, void* workspace, double* stats, int batch, int channels, int t_len, float eps,
                                   void* stream) {
    ACB_REQUIRE(x && workspace && stats, "acb_groupnorm_stats: null pointer");
    ACB_REQUIRE(batch > 0 && batch <= 65535 && channels > 0 && t_len > 0, "acb_groupnorm_stats: bad shape");
    ACB_REQUIRE(eps >= 0.f, "acb_groupnorm_stats: eps < 0");
    const long long n = (long long)channels * t_len;
    const int parts = gn_parts(n);
    cudaStream_t s = (cudaStream_t)stream;
    groupnorm_partial_kernel<<<dim3(parts, batch), GN_THREADS, 0, s>>>(x, (double2*)workspace, n, parts);
    ACB_LAUNCH_CHECK();
    groupnorm_finalize_kernel<<<acb_ceil_div(batch, 8), 256, 0, s>>>(x, (const double2*)workspace, (double2*)stats, n, parts, batch,
                                                                   eps);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

// y = gamma_c (x[left + t] - mean_b) rstd_b + beta_c, plus either a second GroupNorm output of the same shape (the conv shortcut of a
// residual block) or a raw tensor (the identity skip).  x - mean in fp64: the mean can be far larger than the spread.
struct GnApplyParams {
    const float* x; const double2* st; const float* g; const float* be; int t_src, left;
    const float* x2; const double2* st2; const float* g2; const float* be2;
    const float* res; float* y; int C, t_out;
};

__device__ __forceinline__ float gn_norm(float v, double2 st, float g, float be) {
    return fmaf(g * (float)st.y, (float)((double)v - st.x), be);
}

__global__ void __launch_bounds__(256) groupnorm_apply_kernel(GnApplyParams p) {
    const int c = blockIdx.y, b = blockIdx.z;
    const size_t row = (size_t)b * p.C + c;
    const double2 st = p.st[b];
    const float g = p.g[c], be = p.be[c];
    const float* xr = p.x + row * p.t_src + p.left;
    float* yr = p.y + row * p.t_out;
    double2 st2 = make_double2(0.0, 0.0);
    float g2 = 0.f, be2 = 0.f;
    if (p.x2) { st2 = p.st2[b]; g2 = p.g2[c]; be2 = p.be2[c]; }
    const int t0 = blockIdx.x * (256 * 4) + threadIdx.x;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int t = t0 + u * 256;
        if (t >= p.t_out) break;
        float v = gn_norm(__ldg(xr + t), st, g, be);
        if (p.x2) v += gn_norm(__ldg(p.x2 + row * p.t_out + t), st2, g2, be2);
        else if (p.res) v += __ldg(p.res + row * p.t_out + t);
        yr[t] = v;
    }
}

extern "C" int acb_groupnorm_apply(const float* x, const double* stats, const float* gamma, const float* beta, int t_src, int left,
                                   const float* x2, const double* stats2, const float* gamma2, const float* beta2, const float* residual,
                                   float* y, int batch, int channels, int t_out, void* stream) {
    ACB_REQUIRE(x && stats && gamma && beta && y, "acb_groupnorm_apply: null pointer");
    ACB_REQUIRE(batch > 0 && batch <= 65535 && channels > 0 && channels <= 65535 && t_out > 0, "acb_groupnorm_apply: bad shape");
    ACB_REQUIRE(left >= 0 && left + t_out <= t_src, "acb_groupnorm_apply: window [%d, %d) outside %d steps", left, left + t_out, t_src);
    ACB_REQUIRE(!(x2 && residual), "acb_groupnorm_apply: x2 and residual are exclusive");
    ACB_REQUIRE(!x2 || (stats2 && gamma2 && beta2), "acb_groupnorm_apply: x2 needs stats2, gamma2, beta2");
    ACB_REQUIRE(y != x && y != x2 && y != residual, "acb_groupnorm_apply: y must not alias an input");
    GnApplyParams p{x, (const double2*)stats, gamma, beta, t_src, left, x2, (const double2*)stats2, gamma2, beta2, residual, y,
                    channels, t_out};
    groupnorm_apply_kernel<<<dim3(acb_ceil_div(t_out, 256 * 4), channels, batch), 256, 0, (cudaStream_t)stream>>>(p);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}

// ------------------------------------------------------------------------------------------------
// Overlap-add of independently decoded chunks (transformers EncodecModel._linear_overlap_add, as the reference's
// HFEncodecCompressionModel runs the 48 kHz codec): chunk i starts at i*stride, is multiplied by its scale, weighted by the
// triangle w(j) = 0.5 - |(j+1)/(L+1) - 0.5| (L = length of the first chunk) and the sum is divided by the summed weights.
// frames = chunks 0 .. n-2, [n-1][B][C][t_frame]; last = chunk n-1, [B][C][t_last]; scales [n][B] or NULL.
// ------------------------------------------------------------------------------------------------
struct OlaParams {
    const float* frames; const float* last; const float* scales; float* y;
    int n, B, C, t_frame, t_last, stride, t_total, L;
};

__global__ void __launch_bounds__(256) overlap_add_kernel(OlaParams p) {
    const int t = blockIdx.x * 256 + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
    if (t >= p.t_total) return;
    const double inv = 1.0 / (double)(p.L + 1);
    float acc = 0.f, wsum = 0.f;
    for (int i = min(p.n - 1, t / p.stride); i >= 0; --i) {
        const int j = t - i * p.stride;
        const bool is_last = i == p.n - 1;
        if (j >= (is_last ? p.t_last : p.t_frame)) {
            if (j >= p.t_frame) break;   // every earlier chunk ends earlier still
            continue;
        }
        const float w = (float)(0.5 - fabs((double)(j + 1) * inv - 0.5));
        const float v = is_last ? __ldg(p.last + ((size_t)b * p.C + c) * p.t_last + j)
                                : __ldg(p.frames + (((size_t)i * p.B + b) * p.C + c) * p.t_frame + j);
        const float sc = p.scales ? __ldg(p.scales + (size_t)i * p.B + b) : 1.f;
        acc = fmaf(w, v * sc, acc);
        wsum += w;
    }
    p.y[((size_t)b * p.C + c) * p.t_total + t] = acc / wsum;
}

extern "C" int acb_overlap_add(const float* frames, const float* last, const float* scales, float* y, int n_chunks, int batch,
                               int channels, int t_frame, int t_last, int stride, int t_total, void* stream) {
    ACB_REQUIRE(last && y && (n_chunks == 1 || frames), "acb_overlap_add: null pointer");
    ACB_REQUIRE(n_chunks >= 1 && batch > 0 && batch <= 65535 && channels > 0 && channels <= 65535 && stride > 0 && t_last > 0,
                "acb_overlap_add: bad shape");
    ACB_REQUIRE(n_chunks == 1 || (t_frame >= t_last && t_frame >= stride),
                "acb_overlap_add: chunks of %d steps at stride %d leave gaps (last %d)", t_frame, stride, t_last);
    ACB_REQUIRE((long long)stride * (n_chunks - 1) + t_last == t_total, "acb_overlap_add: t_total != stride*(n-1) + t_last");
    OlaParams p{frames, last, scales, y, n_chunks, batch, channels, n_chunks > 1 ? t_frame : t_last, t_last, stride, t_total,
                n_chunks > 1 ? t_frame : t_last};
    overlap_add_kernel<<<dim3(acb_ceil_div(t_total, 256), channels, batch), 256, 0, (cudaStream_t)stream>>>(p);
    ACB_LAUNCH_CHECK();
    return ACB_OK;
}
