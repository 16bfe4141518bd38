// T5 encoder for H100 (sm_90a): transformers' T5EncoderModel forward (the frozen text encoder of T5Conditioner,
// audiocraft/modules/conditioners.py:422-515) followed by the conditioner's output_proj and mask.
//
// A bidirectional pre-norm transformer over the token matrix (M = batch * T rows), on the same machinery as the LM forward:
//   * every matrix product is the tiled wgmma GEMM of fwd_gemm.cuh on the TF32 tensor pipe: fp32 operands in HBM, staged by
//     TMA, fp32 accumulation, no split-K.  Every operand is rounded to the nearest TF32 value before the GEMM reads it (the
//     weights once by the host, the activations by the kernel that writes them) instead of truncated by the tensor core.  fp32 operands keep T5's activation range (pretrained T5's feed-forward activations
//     exceed fp16's 65504) at the same 10-bit mantissa fp16 would have.
//   * epilogues: q / k / v head-major fp16 (the attention kernel's operands), x += acc, ReLU to fp32, and the projection
//     (acc + bias) * mask into the fp32 output.
//   * attention is lm_fwd_attn_kernel<FA_T5> (fwd_attn.cuh): scale 1, the relative-position bias of block 0 shared by every
//     layer, padded keys excluded.
//   * embedding gather and RMSNorm (T5LayerNorm: w * x * rsqrt(mean(x^2) + eps), no mean, no bias) in fp32.
// Stateless and graph-capturable; the caller owns every buffer.
#include "common.cuh"
#include "fwd_attn.cuh"
#include "fwd_gemm.cuh"
#include "lm_math.cuh"
#include <math.h>

// x[m] = shared[ids[m]] (fp32, no scaling, no positional term)
__global__ void __launch_bounds__(256) t5_embed_kernel(const float* __restrict__ shared, const int64_t* __restrict__ ids,
                                                       float* __restrict__ x, int d) {
    const int m = blockIdx.x;
    const float4* src = reinterpret_cast<const float4*>(shared + (size_t)ids[m] * d);
    float4* dst = reinterpret_cast<float4*>(x + (size_t)m * d);
    for (int i = threadIdx.x; i < (d >> 2); i += 256) dst[i] = src[i];
}

// out[m] = w * x[m] * rsqrt(mean(x[m]^2) + eps) rounded to TF32 (the next GEMM's operand); the unrounded fp32 values also into
// out2 when given.  One CTA per row, one float4 per thread.
constexpr int T5_NORM_THREADS = 512;
__global__ void __launch_bounds__(T5_NORM_THREADS) t5_rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                                     float* __restrict__ out, float* __restrict__ out2, int d,
                                                                     float eps) {
    __shared__ float red[32];
    const int r = blockIdx.x, i = threadIdx.x;
    const bool live = i < (d >> 2);
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), g = a;
    if (live) {
        a = reinterpret_cast<const float4*>(x + (size_t)r * d)[i];
        g = reinterpret_cast<const float4*>(w)[i];
    }
    float q = 0.f;
    q = fmaf(a.x, a.x, q); q = fmaf(a.y, a.y, q); q = fmaf(a.z, a.z, q); q = fmaf(a.w, a.w, q);
    const float rs = rsqrtf(block_sum(q, red) / d + eps);
    if (live) {
        const float4 y = make_float4(g.x * (a.x * rs), g.y * (a.y * rs), g.z * (a.z * rs), g.w * (a.w * rs));
        reinterpret_cast<float4*>(out + (size_t)r * d)[i] =
            make_float4(tf32_round(y.x), tf32_round(y.y), tf32_round(y.z), tf32_round(y.w));
        if (out2) reinterpret_cast<float4*>(out2 + (size_t)r * d)[i] = y;
    }
}

namespace {
struct T5Layout {
    size_t x, h, q, k, v, a, f, total;
};

size_t t5_take(size_t* off, size_t bytes) {
    const size_t at = *off;
    *off += (bytes + 255) / 256 * 256;
    return at;
}

// Validates the shapes (no pointer is touched) and lays out the workspace.
int t5_layout(const acb_t5_config* c, int batch, int seq_len, T5Layout* L) {
    ACB_REQUIRE(c, "acb_t5_encode: null config");
    ACB_REQUIRE(c->d_kv == 64, "acb_t5_encode: d_kv %d: the attention kernel is built for 64 (t5-3b / t5-11b use 128)", c->d_kv);
    ACB_REQUIRE(c->d_model >= 64 && c->d_model % 64 == 0 && c->d_model <= 4 * T5_NORM_THREADS,
                "acb_t5_encode: d_model %d must be a multiple of 64 and <= %d (one float4 per RMSNorm thread)", c->d_model,
                4 * T5_NORM_THREADS);
    ACB_REQUIRE(c->num_heads * 64 == c->d_model, "acb_t5_encode: num_heads %d * d_kv 64 must equal d_model %d", c->num_heads,
                c->d_model);
    ACB_REQUIRE(c->num_layers >= 1 && c->d_ff >= 4 && c->d_ff % 4 == 0 && c->vocab_size >= 1 && c->num_buckets >= 1,
                "acb_t5_encode: num_layers %d, d_ff %d (a positive multiple of 4), vocab_size %d, num_buckets %d", c->num_layers,
                c->d_ff, c->vocab_size, c->num_buckets);
    ACB_REQUIRE(c->out_dim >= 2 && c->out_dim % 4 == 0, "acb_t5_encode: out_dim %d must be a positive multiple of 4", c->out_dim);
    ACB_REQUIRE(batch >= 1 && seq_len >= 1, "acb_t5_encode: batch %d, seq_len %d", batch, seq_len);
    const int64_t M = (int64_t)batch * seq_len;
    // the GEMM grid's y dimension is one CTA per FG_BM rows, the embedding / norm grids one CTA per row, the attention grid's
    // z dimension one CTA per item
    constexpr int64_t max_rows = (int64_t)65535 * FG_BM;
    ACB_REQUIRE(M <= max_rows && batch <= 65535,
                "acb_t5_encode: %lld token rows (batch %d): at most %lld rows and 65535 items", (long long)M, batch,
                (long long)max_rows);
    const size_t d = c->d_model, Mz = (size_t)M;
    size_t off = 0;
    L->x = t5_take(&off, Mz * d * 4);
    L->h = t5_take(&off, Mz * d * 4);
    L->q = t5_take(&off, Mz * d * 2);
    L->k = t5_take(&off, Mz * d * 2);
    L->v = t5_take(&off, Mz * d * 2);
    L->a = t5_take(&off, Mz * d * 4);
    L->f = t5_take(&off, Mz * (size_t)c->d_ff * 4);
    L->total = off;
    return ACB_OK;
}
}   // namespace

extern "C" int64_t acb_t5_workspace_bytes(const acb_t5_config* cfg, int batch, int seq_len) {
    T5Layout L;
    const int rc = t5_layout(cfg, batch, seq_len, &L);
    return rc != ACB_OK ? (int64_t)rc : (int64_t)L.total;
}

extern "C" int acb_t5_encode(const acb_t5_config* cfg, const acb_t5_weights* w, const int64_t* ids, const int64_t* mask,
                             const int32_t* buckets, int batch, int seq_len, float* out, float* hidden, void* workspace,
                             int64_t workspace_bytes, void* stream) {
    T5Layout L;
    ACB_TRY(t5_layout(cfg, batch, seq_len, &L));
    const acb_t5_config& c = *cfg;
    ACB_REQUIRE(w && ids && mask && buckets && out && workspace, "acb_t5_encode: null weights, ids, mask, buckets, out or workspace");
    ACB_REQUIRE(w->shared && w->w_qkv && w->w_o && w->w_i && w->w_fo && w->ln && w->final_ln && w->rel_bias && w->proj_w &&
                w->proj_b, "acb_t5_encode: a weight is NULL");
    ACB_REQUIRE(workspace_bytes >= (int64_t)L.total, "acb_t5_encode: workspace of %lld bytes < %lld needed",
                (long long)workspace_bytes, (long long)L.total);
    cudaStream_t s = (cudaStream_t)stream;
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    float *x = reinterpret_cast<float*>(ws + L.x), *h = reinterpret_cast<float*>(ws + L.h);
    float *a = reinterpret_cast<float*>(ws + L.a), *f = reinterpret_cast<float*>(ws + L.f);
    __half *q = reinterpret_cast<__half*>(ws + L.q), *k = reinterpret_cast<__half*>(ws + L.k), *v = reinterpret_cast<__half*>(ws + L.v);
    const int d = c.d_model, ff = c.d_ff, H = c.num_heads, NL = c.num_layers, T = seq_len, M = batch * T;

    // tensor maps: fp32 activations [rows][K] and stacked fp32 weights [L * N][K], 128-row boxes
    CUtensorMap m_h, m_a, m_f, m_qkv, m_o, m_i, m_fo, m_proj;
    ACB_TRY(encode_map_f32(&m_h, h, d, M, FG_BM));
    ACB_TRY(encode_map_f32(&m_a, a, d, M, FG_BM));
    ACB_TRY(encode_map_f32(&m_f, f, ff, M, FG_BM));
    ACB_TRY(encode_map_f32(&m_qkv, w->w_qkv, d, NL * 3 * d, FG_BN));
    ACB_TRY(encode_map_f32(&m_o, w->w_o, d, NL * d, FG_BN));
    ACB_TRY(encode_map_f32(&m_i, w->w_i, d, NL * ff, FG_BN));
    ACB_TRY(encode_map_f32(&m_fo, w->w_fo, ff, NL * d, FG_BN));
    ACB_TRY(encode_map_f32(&m_proj, w->proj_w, d, c.out_dim, FG_BN));

    t5_embed_kernel<<<M, 256, 0, s>>>(w->shared, ids, x, d);
    ACB_LAUNCH_CHECK();
    FwdGemmParams base{};
    base.M = M; base.K = d; base.T = T; base.H = H; base.d = d;
    base.q = q; base.k = k; base.v = v; base.x = x; base.f32 = f;
    auto norm = [&](const float* gamma, float* out2) -> int {
        t5_rmsnorm_kernel<<<M, T5_NORM_THREADS, 0, s>>>(x, gamma, h, out2, d, c.eps);
        ACB_LAUNCH_CHECK();
        return ACB_OK;
    };
    FwdAttnParams at{};
    at.q = q; at.k = k; at.v = v; at.H = H; at.Tq = T; at.Tk = T; at.d = d; at.scale = 1.f;
    at.out32 = a; at.rel_bias = w->rel_bias; at.buckets = buckets; at.key_mask = mask;
    const dim3 agrid(acb_ceil_div(T, FA_BQ), H, batch);
    for (int l = 0; l < NL; ++l) {
        // self attention
        ACB_TRY(norm(w->ln + (size_t)l * 2 * d, nullptr));
        FwdGemmParams p = base;
        p.N = 3 * d; p.w_row0 = l * 3 * d;
        ACB_TRY((fwd_gemm<FE_QKV, true>(m_h, m_qkv, p, s)));
        lm_fwd_attn_kernel<FA_T5><<<agrid, 128, 0, s>>>(at);
        ACB_LAUNCH_CHECK();
        p = base;
        p.N = d; p.w_row0 = l * d;
        ACB_TRY((fwd_gemm<FE_RESID, true>(m_a, m_o, p, s)));
        // feed forward: x += wo(relu(wi(norm(x))))
        ACB_TRY(norm(w->ln + ((size_t)l * 2 + 1) * d, nullptr));
        p = base;
        p.N = ff; p.w_row0 = l * ff;
        ACB_TRY((fwd_gemm<FE_RELU, true>(m_h, m_i, p, s)));
        p = base;
        p.N = d; p.K = ff; p.w_row0 = l * d;
        ACB_TRY((fwd_gemm<FE_RESID, true>(m_f, m_fo, p, s)));
    }
    ACB_TRY(norm(w->final_ln, hidden));
    FwdGemmParams p = base;
    p.N = c.out_dim; p.w_row0 = 0; p.f32 = out; p.bias = w->proj_b; p.mask = mask;
    return fwd_gemm<FE_PROJ, true>(m_h, m_proj, p, s);
}
