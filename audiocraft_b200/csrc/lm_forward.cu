// MusicGen LM full-sequence forward for H100 (sm_90a): LMModel.forward over whole sequences (audiocraft/models/lm.py:221-268),
// the computation behind LMModel.compute_predictions (lm.py:270-321), i.e. scoring codes under the LM.
//
// Unlike the decode step (lm.cu), which streams every weight once per generated position and is bound by HBM bandwidth, the
// forward multiplies the whole token matrix (M = batch * (prefix + seq_len) rows) by each weight once and is compute-bound:
//   * every matrix product is one tiled wgmma GEMM (lm_fwd_gemm_kernel, fwd_gemm.cuh): 128 x 128 output tiles, both operands K-major in
//     the 128-byte swizzle that tiled TMA writes into an mbarrier ring, one producer warp issuing the loads and two consumer
//     warpgroups issuing the MMAs.  No split-K: every output element is summed by one CTA in one fixed order, so an item's
//     results do not depend on the batch it is in, and the residual add is a plain read-modify-write.
//   * the epilogue of each GEMM writes its consumer's layout directly: q / k / v head-major (with rotary positions), the
//     condition's cross K / V, x += acc, GELU to fp16, or fp32 logits of the sequence positions.
//   * attention is a flash-attention kernel on mma.sync (lm_fwd_attn_kernel, fwd_attn.cuh): causal for self attention, every text position
//     (padding included, as the reference does) for cross attention.
// fp16 GEMM operands, fp32 accumulation, fp32 residual stream and LayerNorm, as in the decode step (DESIGN.md section 2).
// The kernels restate the element arithmetic of the decode kernels (embedding + sin term, LayerNorm, GELU, rotary) so that
// forward and decode agree.  Nothing here touches a decode handle: the call is stateless and graph-capturable.
#include "common.cuh"
#include "fwd_attn.cuh"
#include "fwd_gemm.cuh"
#include "lm_math.cuh"
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

int fwd_attn(bool causal, const FwdAttnParams& a, int batch, cudaStream_t s) {
    const dim3 grid(acb_ceil_div(a.Tq, FA_BQ), a.H, batch);
    if (causal) lm_fwd_attn_kernel<FA_CAUSAL><<<grid, 128, 0, s>>>(a);
    else lm_fwd_attn_kernel<FA_CROSS><<<grid, 128, 0, s>>>(a);
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
