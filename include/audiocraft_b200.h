/*
 * audiocraft_b200 -- C-ABI of the H100 (sm_90a) hot-path library.
 *
 * The reference (facebookresearch/audiocraft) is 100% Python and has no FFI layer; its boundary for
 * this path is the Python class API (CompressionModel / LMModel / MusicGen).  This header is the
 * boundary a native replacement exports underneath those classes; each entry point cites the
 * reference function it replaces (paths relative to the reference repo root).  INTEGRATION.md shows
 * the ctypes stub a maintainer adds on the reference side.
 *
 * Conventions
 *   - every function returns 0 on success, a negative acb_status otherwise; acb_last_error() gives
 *     a human readable message for the calling thread.  No C++ exception crosses the ABI.
 *   - all pointers are DEVICE pointers unless named host_*; the caller (PyTorch) owns every buffer,
 *     including KV caches and workspaces.  The library allocates nothing after acb_lm_create().
 *   - all work is enqueued on the caller's CUDA stream (`stream` is a cudaStream_t passed as void*),
 *     nothing synchronises the device, so every call is CUDA-graph capturable unless noted.
 *   - handles are not thread-safe; one handle per device.
 *   - tensors are dense row-major; "BCT" means [batch][channel][time] float32.
 */
#ifndef AUDIOCRAFT_B200_H
#define AUDIOCRAFT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    ACB_OK = 0,
    ACB_ERR_INVALID = -1,     /* bad argument / unsupported shape */
    ACB_ERR_CUDA = -2,        /* a CUDA runtime call failed */
    ACB_ERR_UNSUPPORTED = -3, /* valid in the reference, not built here (say which in last_error) */
} acb_status;

int acb_version(void);
const char* acb_last_error(void);
/* Device properties the host side sizes its launches with. */
int acb_device_sm_count(int device);

/* ---------------------------------------------------------------- EnCodec: SEANet convolutions ---- */

/* w[g][i] = g[g] * v[g][i] / ||v[g]||_2   (one warp-shuffle reduction per group).
 * Replaces the weight_norm forward pre-hook that audiocraft/modules/conv.py:21-30 installs and that
 * recomputes the weight on EVERY forward; here it is folded once at load.  groups = dim 0 of the
 * parameter (Cout for Conv1d, Cin for ConvTranspose1d), inner = product of the other dims. */
int acb_weight_norm_fold(const float* v, const float* g, float* w, int groups, int inner, void* stream);

/* StreamableConv1d.forward, audiocraft/modules/conv.py:185-201, with the padding folded into index
 * math (no F.pad copy) and the surrounding elementwise ops fused:
 *   y[b,co,t] = bias[co] + sum_{ci,k} w[ci*K+k][co] * act(xpad[b,ci,t*stride + k*dilation - pad_left])
 *               (+ residual[b,co,t])
 *   act = ELU(alpha=1) if elu_in else identity  (the nn.ELU that precedes the conv, seanet.py:45,131,143)
 *   xpad = reflect (reflect=1; with the short-input rule of conv.py:71-88: virtual length t_virtual >= t_in,
 *          zeros past t_in) or zero padding (reflect=0) of x; pad_left / t_out come from the host, which
 *          mirrors get_extra_padding_for_conv1d (conv.py:47-53).
 *   residual: the true-skip input of SEANetResnetBlock (seanet.py:59-60), or NULL.
 * w_packed is [Cin*K][Cout] (tap-major, Cout contiguous), folded fp32 weights. */
int acb_conv1d(const float* x, const float* w_packed, const float* bias, const float* residual, float* y,
               int batch, int c_in, int c_out, int t_in, int t_virtual, int t_out, int kernel, int stride,
               int dilation, int pad_left, int reflect, int elu_in, int precision, void* stream);
/* precision: ACB_CONV_FP32 = fp32 FMA (what the RVQ-exact encoder uses); ACB_CONV_TF32X3 = tensor pipe with every fp32
 * operand split into two tf32 terms and three MMAs per product (~2^-22 relative error per product, fp32 accumulate) --
 * layers too small for the MMA tile fall back to fp32 FMA. */
#define ACB_CONV_FP32 0
#define ACB_CONV_TF32X3 1          /* wgmma tf32 (3xTF32 split), accumulator in registers */
#define ACB_CONV_TF32X3_MMASYNC 2  /* same arithmetic on the legacy mma.sync.m16n8k8 path */

/* StreamableConvTranspose1d.forward, audiocraft/modules/conv.py:221-243: transposed conv (kernel = 2*stride)
 * followed by the fixed trim, computed directly in trimmed coordinates:
 *   y[b,co,o] = bias[co] + sum_ci ( act(x[b,ci,ti]) * w[ci][p][co] + act(x[b,ci,ti-1]) * w[ci][p+stride][co] ),
 *   u = o + trim_left, ti = u / stride, p = u % stride, x outside [0,t_in) = 0.
 * w_packed is [Cin][K][Cout].  Supported strides: 2,3,4,5,8 with kernel == 2*stride. */
int acb_convtr1d(const float* x, const float* w_packed, const float* w_gemm, const float* bias, float* y,
                 int batch, int c_in, int c_out, int t_in, int t_out, int kernel, int stride, int trim_left,
                 int elu_in, int precision, void* stream);

/* The encoder's default for k > 1, >= 128 output channels (RVQ indices exact on the 10 s goldens): the same convolution as
 * acb_conv1d (StreamableConv1d.forward, modules/conv.py:185-201, + fused ELU / residual) as an implicit GEMM on wgmma
 * without an im2col tile, the tensor-core accumulator flushed into fp32 registers once per 8 input channels (csrc/encodec.cu,
 * conv1d_t6_kernel).  c_in % 8 == 0 and c_out % 64 == 0.  w6 = weights split into two tf32 terms and laid out as
 * [c_out / N][c_in / 8][kernel][term hi,lo][2][N][4] with N = acb_conv1d_t6_tile(c_out)
 * (audiocraft_b200.encodec.pack_conv_t6 builds it). */
int acb_conv1d_t6(const float* x, const float* w6, const float* bias, const float* residual, float* y, int batch,
                  int c_in, int c_out, int t_in, int t_virtual, int t_out, int kernel, int stride, int dilation,
                  int pad_left, int reflect, int elu_in, void* stream);
int acb_conv1d_t6_tile(int c_out);   /* output-channel tile (128, 64, or 0 = shape not supported) */
/* SEANetResnetBlock.forward with the identity skip (audiocraft/modules/seanet.py:44-69, true_skip=True; one residual layer of
 * kernel sizes [k, 1]) as one kernel:  y = x + conv1x1(elu(conv_k(elu(x)))).  w1 is the first conv's folded weight packed
 * [k][C][C/2] (tap-major), w2 the second conv's packed [C/2][C]; pad_left / reflect as acb_conv1d (stride 1).  Tensor pipe with
 * every fp32 operand split into two fp16 terms (22 mantissa bits; |values| must stay below fp16's 65504), three MMAs per product;
 * exact != 0 bounds every tensor-core accumulation run to 48 (resp. 16) reduction rows with fp32 adds in between
 * (the encoder setting: RVQ indices equal the fp32 reference's).  x and y must not alias. */
int acb_resblock_supported(int channels, int kernel, int dilation);
int acb_resblock(const float* x, const float* w1, const float* b1, const float* w2, const float* b2, float* y, int batch,
                 int channels, int t_len, int kernel, int dilation, int pad_left, int reflect, int exact, void* stream);

/* w_gemm (optional, needed for precision ACB_CONV_TF32X3): the same weights packed as the GEMM operand
 * [2*Cin][Cout*stride], row r = ci*2 + k (k = 0 multiplies x[ti-1], k = 1 multiplies x[ti]), column n' = co*stride + ph,
 * value w[ci][ph + (1-k)*stride][co]: the transposed conv then runs on the tensor-core kernel as one GEMM whose accumulator
 * row ti holds `stride` consecutive output steps of every channel. */

/* Recurrent half of StreamableLSTM.forward, audiocraft/modules/lstm.py:19-25 (nn.LSTM, gate order i,f,g,o,
 * zero initial state).  The input half (W_ih x_t + b_ih + b_hh for every t) is a 1x1 acb_conv1d producing
 * gates_x [B][4H][T]; this call runs the T dependent steps in ONE persistent cooperative kernel that keeps
 * its slice of W_hh resident in shared memory:
 *   y[b,:,t] = h_t (+ skip[b,:,t] if skip != NULL)       [B][H][T]
 * state_ws: acb_lstm_state_bytes(B, H) bytes of scratch = (2*max(B,32)*H + 64) floats (h double buffer, kept for 32 item slots in
 * MMA-fragment order by the tensor-core kernel, + grid-barrier counter), zeroed by the call.  hidden % 64 == 0 and B <= 32 run the
 * recurrent step on the tensor pipe (hidden % 128 == 0: both operands split into two fp16 terms, 22 mantissa bits; else 3xTF32;
 * fp32 accumulate), other shapes on fp32 FMA.
 * NOT graph-capturable (cooperative launch). */
int acb_lstm_recurrent(const float* gates_x, const float* w_hh, const float* skip, float* y, float* state_ws,
                       int batch, int hidden, int t_len, void* stream);
/* bytes of state_ws needed by acb_lstm_recurrent and acb_lstm_recurrent_carry */
int64_t acb_lstm_state_bytes(int batch, int hidden);
/* acb_lstm_recurrent from a carried state, for a sequence decoded in pieces: h_state and c_state are caller-owned [B][H] fp32
 * arrays, read as the state before step 0 and overwritten with the state after step t_len - 1.  Same kernels, same routing and
 * the same operations in the same order: running T = t1 + t2 + ... steps as pieces, with the state carried between the calls,
 * gives y and the final (h, c) bit-identical to one call of T steps.  One more grid barrier than acb_lstm_recurrent publishes
 * the carried h before step 0. */
int acb_lstm_recurrent_carry(const float* gates_x, const float* w_hh, const float* skip, float* y, float* state_ws,
                             float* h_state, float* c_state, int batch, int hidden, int t_len, void* stream);

/* ---------------------------------------------------------------- EnCodec: residual VQ ------------- */

/* ResidualVectorQuantizer.encode, audiocraft/quantization/vq.py:87-96 -> core_vq.py:386-396 -> :164-172,
 * fused per codebook: score_j = -(|r|^2 - 2 r.e_j + |e_j|^2) in fp32, first-max argmax, r -= e_idx.
 * The [frames x bins] distance matrix never goes to HBM.
 *   latent [B][D][T] fp32, codebooks [n_q][bins][D] fp32, cb_sqnorm [n_q][bins] fp32 (sum_d e^2),
 *   codes [B][n_q][T] int64.  D must be a multiple of 4 and <= 512. */
int acb_rvq_encode(const float* latent, const float* codebooks, const float* cb_sqnorm, int64_t* codes,
                   int batch, int dim, int t_len, int n_q, int bins, void* stream);

/* ResidualVectorQuantizer.decode, vq.py:98-103 -> core_vq.py:398-404: latent[b,:,t] = sum_k E_k[codes[b,k,t]]. */
int acb_rvq_decode(const int64_t* codes, const float* codebooks, float* latent,
                   int batch, int dim, int t_len, int n_q, int bins, void* stream);

/* ---------------------------------------------------------------- EnCodec: GroupNorm, chunking ----- */

/* Statistics of GroupNorm(1, C) (norm='time_group_norm', audiocraft/modules/conv.py:33-42) over each item of x [B][C][T]:
 * stats[b] = {mean, 1/sqrt(var + eps)} as two doubles (biased variance over the C*T elements).  Deterministic: an item's
 * statistics do not depend on the batch it sits in; fp64 sums of x - x[b][0][0], so a large mean does not cancel the variance.
 * workspace: acb_groupnorm_workspace_bytes(B, C, T) bytes of scratch. */
int64_t acb_groupnorm_workspace_bytes(int batch, int channels, int t_len);
int acb_groupnorm_stats(const float* x, void* workspace, double* stats, int batch, int channels, int t_len, float eps, void* stream);

/* y[b,c,t] = gamma[c] (x[b,c,left+t] - mean_b) rstd_b + beta[c] for t in [0, t_out), x being [B][C][t_src] (left > 0 reads the
 * window the transposed conv's trim keeps: NormConvTranspose1d normalises before StreamableConvTranspose1d trims, conv.py:221-243),
 *   + the same normalisation of x2 [B][C][t_out] with stats2 / gamma2 / beta2 (a residual block's conv shortcut), or
 *   + residual [B][C][t_out] (the identity skip); x2 and residual may both be NULL, not both set.  y aliases no input. */
int acb_groupnorm_apply(const float* x, const double* stats, const float* gamma, const float* beta, int t_src, int left,
                        const float* x2, const double* stats2, const float* gamma2, const float* beta2, const float* residual,
                        float* y, int batch, int channels, int t_out, void* stream);

/* Linear overlap-add of the independently decoded chunks of the chunked (48 kHz) codec, transformers
 * EncodecModel._linear_overlap_add: chunk i starts at i*stride, is multiplied by scales[i][b] (scales NULL: 1), weighted by the
 * triangle w(j) = 0.5 - |(j+1)/(L+1) - 0.5| with L the first chunk's length, and the weighted sum is divided by the summed weights.
 * frames: chunks 0 .. n-2 as [n-1][B][C][t_frame] (NULL when n_chunks == 1); last: chunk n-1 as [B][C][t_last];
 * y [B][C][t_total], t_total = stride*(n_chunks-1) + t_last. */
int acb_overlap_add(const float* frames, const float* last, const float* scales, float* y, int n_chunks, int batch, int channels,
                    int t_frame, int t_last, int stride, int t_total, void* stream);

/* ---------------------------------------------------------------- MusicGen: LM decode -------------- */

typedef struct {
    int dim;          /* d_model */
    int num_heads;    /* head_dim must be 64 */
    int num_layers;
    int ffn_dim;      /* hidden_scale * dim */
    int n_q;          /* codebooks (4) */
    int card;         /* cardinality (2048); special token id == card */
    int cross_attention; /* 1: layers have cross attention to the text condition */
    int max_rows;     /* rows = B (no CFG) or 2B (CFG: [cond rows; null rows]) the buffers are sized for, 1 .. ACB_LM_MAX_ROWS.
                         Up to 64 rows every GEMM of the step is the mma.sync kernel; above 64 rows the wgmma kernel
                         (lm_gemm_wide_kernel), which needs ffn_dim and n_q * card to be multiples of 64 (else acb_lm_begin
                         returns ACB_ERR_UNSUPPORTED) */
    int max_seq;      /* S = T + max_delay + 1, KV cache length */
    int max_text;     /* cross-attention source length the cross KV cache is sized for */
    float pos_scale;  /* positional_scale */
    int positional_embedding; /* 0 'sin' (released MusicGen), 1 'rope', 2 'sin_rope'  (modules/transformer.py:632-637, 701-705).
                                 rope and sin_rope need weights.rope_freq */
    int weight_dtype; /* the seven per-layer matrices w_qkv .. w_ff2: 0 fp16; 1 e4m3 codes (one byte each, same [L][N][K]
                         layout) with one fp32 scale per output row in s_qkv .. s_ff2, W[n][k] = code[n][k] * scale[n] with
                         scale = amax_k |W[n][k]| / 448 (see audiocraft_b200.lm.quantize_rows_e4m3).  The decode GEMMs unpack
                         the codes exactly to fp16, accumulate code x activation in fp32 and multiply each output's sum by its
                         row scale once; acb_lm_forward dequantizes one layer at a time into its workspace.  emb, heads and
                         the norms stay as they are.  acb_lm_create / acb_lm_forward return ACB_ERR_INVALID when a scale the
                         model needs is NULL or the value is neither 0 nor 1. */
} acb_lm_config;

/* fp16 matrices in the reference's own [out_features][in_features] layout, stacked over layers (the seven per-layer
 * matrices as e4m3 codes in the same layout when acb_lm_config.weight_dtype is 1). */
typedef struct {
    const void* emb;      /* [n_q][card+1][d] fp16       LMModel.emb, lm.py:160-163 */
    const float* inv_freq;/* [d/2] fp32: max_period^(i/(d/2-1)), create_sin_embedding transformer.py:70-89 */
    const void* w_qkv;    /* [L][3d][d]   self_attn.in_proj_weight (packed p,h,hd; transformer.py:373) */
    const void* w_o;      /* [L][d][d]    self_attn.out_proj.weight */
    const void* w_cq;     /* [L][d][d]    cross_attention.in_proj_weight[:d] */
    const void* w_ckv;    /* [L][2d][d]   cross_attention.in_proj_weight[d:] */
    const void* w_co;     /* [L][d][d]    cross_attention.out_proj.weight */
    const void* w_ff1;    /* [L][ffn][d]  linear1.weight */
    const void* w_ff2;    /* [L][d][ffn]  linear2.weight */
    const float* ln;      /* [L][6][d] fp32: norm1.w, norm1.b, norm_cross.w, norm_cross.b, norm2.w, norm2.b */
    const float* out_norm;/* [2][d] fp32 */
    const void* heads;    /* [n_q*card][d] fp16  LMModel.linears, lm.py:172 */
    const float* rope_freq; /* [32] fp32: 1 / max_period^(2i/64), RotaryEmbedding.frequencies rope.py:68-69 (NULL without rope) */
    /* weight_dtype 1 only (NULL otherwise): fp32 row scales of w_qkv .. w_ff2, [L][N] with N their output features
       (3d, d, d, 2d, d, ffn, d); s_cq, s_ckv and s_co are needed only with cross attention */
    const float* s_qkv;
    const float* s_o;
    const float* s_cq;
    const float* s_ckv;
    const float* s_co;
    const float* s_ff1;
    const float* s_ff2;
} acb_lm_weights;

/* Caller-owned state; sizes in elements.  rows_pad = acb_lm_rows_pad(max_rows) (a multiple of 16). */
typedef struct {
    float* x;          /* [rows_pad][d]            residual stream */
    void* h16;         /* [rows_pad][d] fp16       LayerNorm output / GEMM input */
    void* a16;         /* [rows_pad][d] fp16       attention output */
    void* f16;         /* [rows_pad][ffn] fp16     gelu(linear1) */
    float* q32;        /* [rows_pad][d]            self-attention queries */
    float* part;       /* [ACB_LM_PART_SLOTS][rows_pad][max(3d, ffn, n_q*card)]  split-K partial sums */
    float* logits;     /* [rows_pad][n_q*card] */
    void* k_cache;     /* [L][max_rows][H][max_seq][64] fp16; NULL (with v_cache) for a paged handle (acb_lm_begin_slots_paged) */
    void* v_cache;     /* same */
    void* ck_cache;    /* [L][max_rows][H][max_text][64] fp16  cross-attention keys (computed once per generate) */
    void* cv_cache;    /* same, values */
    void* cross16;     /* [max_rows*max_text rounded up to 64][d] fp16  staging of the condition tensor */
    int64_t* seq;      /* [B][n_q][max_seq]  delay-pattern sequence, -1 = not generated yet */
    uint8_t* seq_mask; /* [n_q][max_seq]     pattern validity mask (codebooks_patterns.py:130-152) */
    int32_t* pos;      /* [4] device ints: pos (tokens in the KV cache), rows, batch, text_len */
    float* noise;      /* [B][n_q][card] Exponential(1) noise, read when sampling.noise_from_buffer != 0 */
    /* slot mode only (acb_lm_begin_slots; NULL otherwise), with B = slots in seq above: */
    int32_t* slot_sampling; /* [slots][ACB_LM_SLOT_SAMPLING_STRIDE] 32-bit words per slot: use_sampling, temp (fp32 bits), top_k,
                               top_p (fp32 bits), cfg_coef (fp32 bits), 3 unused (written by the library at admission) */
    int32_t* slot_state; /* [slots][ACB_LM_SLOT_STRIDE] per-slot position, status, lengths, seed and condition-prefix length
                            (written by the library) */
    uint8_t* slot_mask;  /* [slots][n_q][max_seq] each slot's pattern validity mask (written by the caller before acb_lm_admit) */
} acb_lm_buffers;

#define ACB_LM_SLOT_STRIDE 8     /* int32 words of slot_state per slot */
#define ACB_LM_SLOT_SAMPLING_STRIDE 8   /* 32-bit words of slot_sampling per slot */
#define ACB_LM_MAX_SLOTS 128     /* slots of a session: rows = 2 * slots <= ACB_LM_MAX_ROWS */
#define ACB_LM_MAX_SPLIT 8
#define ACB_LM_PART_SLOTS 16
#define ACB_LM_PREFILL_ROWS 64   /* (token, row) pairs one prefill pass handles = the tallest GEMM tile; above 64 rows a pass
                                    holds one position of every row */
#define ACB_LM_MAX_ROWS 256      /* rows one handle decodes: the widest wgmma tile (N = 256) */
#define ACB_LM_KV_PAGE 64        /* cache positions per page of a paged slot session (acb_lm_begin_slots_paged): a multiple of
                                    the 4-position groups the attention kernel copies, so no 16-byte copy crosses a page */
#define ACB_LM_MAX_PAGES_PER_ROW 188   /* ceil(12000 / ACB_LM_KV_PAGE): pages of one row at the largest max_seq */

typedef struct {
    int use_sampling;  /* LMModel.generate(use_sampling, temp, top_k, top_p, cfg_coef), lm.py:421-436 */
    float temp;
    int top_k;
    float top_p;
    float cfg_coef;
    uint64_t seed;     /* Philox key for the on-device sampler */
    int noise_from_buffer; /* 1: take the Exponential(1) noise from acb_lm_buffers.noise / the `noise` argument
                              (parity tests inject torch's stream); 0: on-device Philox */
    float cfg_coef_beta;   /* double CFG (MusicGen-Style, lm.py:362-376), used when rows == 3*batch = [cond; style-only; null]:
                              logits = null + cfg_coef * (style + cfg_coef_beta * (cond - style) - null) */
} acb_lm_sampling;

typedef struct acb_lm acb_lm_t;

int acb_lm_create(const acb_lm_config* cfg, const acb_lm_weights* w, const acb_lm_buffers* buf, acb_lm_t** out);
int acb_lm_destroy(acb_lm_t* lm);

/* Start a generation: rows = batch (cross == NULL or cfg disabled) or 2*batch (CFG).  cross is the fp32
 * condition tensor [rows][text_len][d] the reference's fuser hands to the transformer as
 * cross_attention_src (conditioners.py:1731-1746; padded / null positions are exact zeros and are still
 * attended to).  Computes every layer's cross K/V ONCE (the reference recomputes them every step,
 * transformer.py:355-357), resets pos to 0 and captures the per-step CUDA graph. */
int acb_lm_begin(acb_lm_t* lm, const float* cross, int batch, int rows, int text_len, int seq_len,
                 const acb_lm_sampling* sampling, void* stream);

/* acb_lm_begin for a model whose fuser prepends conditions to the token embeddings (`prepend`, MusicGen-melody;
 * conditioners.py:1703-1763).  prefix is fp32 [rows][prefix_len][d], one prefix per row (cond and null rows differ); each value
 * is rounded to fp16 on the device, as the reference's autocast output_proj rounds it.  The prefix fills KV-cache positions
 * [0, prefix_len) once, in prefill passes (every layer, cross attention included when the model has it); afterwards sequence
 * column t runs at cache position prefix_len + t, for decode steps and acb_lm_prefill alike, while acb_lm_prefill still takes
 * sequence columns.  Needs prefix_len + seq_len <= max_seq; any rows up to max_rows (above ACB_LM_PREFILL_ROWS the passes
 * hold one prefix position of every row).  prefix_len == 0 is acb_lm_begin. */
int acb_lm_begin_prefix(acb_lm_t* lm, const float* cross, const float* prefix, int prefix_len, int batch, int rows,
                        int text_len, int seq_len, const acb_lm_sampling* sampling, void* stream);

/* n_steps iterations of the hot loop of LMModel.generate (lm.py:540-565): for the current offset = pos+1,
 * feed seq[:,:,pos], run the transformer (LMModel.forward lm.py:221-268), CFG-mix, sample
 * (_sample_next_token lm.py:393-418), apply the pattern mask and write seq[:,:,offset] where it is still -1.
 * Each step is one CUDA-graph launch; nothing returns to the host. */
int acb_lm_steps(acb_lm_t* lm, int n_steps, void* stream);

/* Prompt prefill = the reference's multi-token first call (modules/transformer.py:240-247, 413-414; models/lm.py:513-534):
 * consume sequence positions [pos0, pos0 + n_tokens) of every row -- their tokens are already in buffers.seq -- without
 * sampling, ACB_LM_PREFILL_ROWS / rows positions per pass (the per-phase kernels on (token, row) pairs, causal inside a pass;
 * one position per pass above ACB_LM_PREFILL_ROWS rows), and leave the device position at pos0 + n_tokens.  The activation
 * buffers must hold max(ACB_LM_PREFILL_ROWS, acb_lm_rows_pad(rows)) rows. */
int acb_lm_prefill(acb_lm_t* lm, int pos0, int n_tokens, void* stream);

/* Slot mode (continuous batching): a session of `slots` independent requests in the CFG layout, slot s owning rows s (cond)
 * and slots + s (null), rows = 2 * slots <= max_rows, 1 <= slots <= ACB_LM_MAX_SLOTS.  Requests enter free slots between
 * steps (acb_lm_admit) and leave when their last column is sampled, while the other slots keep decoding; every slot has its
 * own position, sequence length, text length and seed.  The GEMMs run on all rows whichever slots are busy, so their regime
 * and K split are fixed for the session.  Each slot attends to exactly its own text length, and its noise is Philox stream k
 * of (its seed, column) -- what acb_lm_begin draws for item 0 -- so a request's tokens are those of the same request
 * generated alone (bit for bit where both run the same GEMM regime, i.e. up to 64 rows).  Needs buffers.slot_sampling,
 * buffers.slot_state and buffers.slot_mask.  `sampling` holds the session's default options, which a request admitted without
 * its own takes; cfg_coef_beta != 0 returns ACB_ERR_UNSUPPORTED and noise_from_buffer is refused.  Marks every slot inactive
 * and captures the session's step graph, which acb_lm_steps then launches.
 * max_text <= max_text of the config bounds the admitted conditions, seq_len_max <= max_seq their sequences. */
int acb_lm_begin_slots(acb_lm_t* lm, int slots, int max_text, int seq_len_max, const acb_lm_sampling* sampling, void* stream);

/* Admit a request into `slot` (free: never used, finished or retired) between steps: writes the slot's cross-attention K/V from
 * cross, the fp32 condition [2][text_len][d] ([cond; null] rows, NULL without cross attention), and starts the slot at column 0
 * with sequence length seq_len and the Philox key seed.  The caller first writes the slot's delay-pattern sequence into
 * buffers.seq[slot] (-1 where unknown; known prompt tokens are kept and consumed one column per step) and its mask into
 * buffers.slot_mask[slot].  After seq_len - 1 steps the slot has written column seq_len - 1 and is finished.
 * sampling: the request's own use_sampling, temp, top_k, top_p and cfg_coef, written to buffers.slot_sampling[slot], where the
 * captured step reads them (slots with different options share one step); NULL takes the options of acb_lm_begin_slots.  seed,
 * noise_from_buffer and cfg_coef_beta of the struct: seed is the argument above, noise_from_buffer != 0 and cfg_coef_beta != 0
 * are refused (ACB_ERR_INVALID, ACB_ERR_UNSUPPORTED).  Needs temp >= 0, top_k >= 0, 0 <= top_p <= 1 and a finite cfg_coef
 * (else ACB_ERR_INVALID); as in acb_lm_begin, top_p > 0 samples top-p, else top_k > 0 top-k, and use_sampling == 0 or
 * temp == 0 takes the argmax. */
int acb_lm_admit(acb_lm_t* lm, int slot, const float* cross, int text_len, int seq_len, uint64_t seed,
                 const acb_lm_sampling* sampling, void* stream);

/* acb_lm_admit for a model whose fuser prepends conditions (`prepend`, MusicGen-melody): prefix is the request's fp32
 * [2][prefix_len][d] ([cond; null] rows), which fills cache positions [0, prefix_len) of the slot's two rows, after the
 * cross K/V, in the prefill passes acb_lm_begin_prefix runs for a generation of batch 1 with CFG (ACB_LM_PREFILL_ROWS / 2
 * positions per pass), so the K/V are the ones that generation writes.  The slot then runs column t at cache position
 * prefix_len + t; its position (acb_lm_slot_status) still counts columns.  Every slot has its own prefix length.  Writes only
 * the slot's cache rows, sequence row, mask, sampling record and state; the passes use the activation buffers and
 * buffers.pos, which the session's step does not carry between steps, and leave the session's padded activation rows zero.
 * Needs prefix_len >= 0, a prefix when prefix_len > 0 and prefix_len + seq_len <= max_seq (else ACB_ERR_INVALID, before
 * anything is enqueued).  prefix_len == 0 is acb_lm_admit. */
int acb_lm_admit_prefix(acb_lm_t* lm, int slot, const float* cross, int text_len, const float* prefix, int prefix_len,
                        int seq_len, uint64_t seed, const acb_lm_sampling* sampling, void* stream);

/* Paged slot session: acb_lm_begin_slots with the self-attention KV cache in a pool of pages instead of `slots` rows of
 * max_seq positions, so a request holds only the pages its own length needs.  Only on a handle created with
 * buffers.k_cache = buffers.v_cache = NULL (a paged handle; acb_lm_begin, acb_lm_begin_prefix, acb_lm_prefill and
 * acb_lm_begin_slots return ACB_ERR_INVALID on it, and this call returns it on any other handle).
 *   k_pool, v_pool  fp16 [L][n_pages][H][ACB_LM_KV_PAGE][64]: page j of a row holds its cache positions
 *                   [ACB_LM_KV_PAGE * j, ACB_LM_KV_PAGE * (j + 1)).
 *   page_table      int32 [2 * slots][pages_per_row] (device): row r's page ids, written by acb_lm_admit_paged for the
 *                   slot's two rows; the captured step reads it at run time, so an admission recaptures nothing.
 *                   ceil((max_prefix + seq_len_max) / ACB_LM_KV_PAGE) <= pages_per_row <= ACB_LM_MAX_PAGES_PER_ROW.
 *   stage_k, stage_v  fp16 [L][2][H][max_prefix][64]: an admission runs a condition prefix's prefill passes into these
 *                   (the passes acb_lm_admit_prefix runs) and copies them into the slot's pages; NULL when max_prefix == 0.
 * Needs max_prefix + seq_len_max <= max_seq and n_pages >= 2 * ceil((max_prefix + seq_len_max) / ACB_LM_KV_PAGE) (one
 * request of the longest length fits).  Everything else is acb_lm_begin_slots. */
int acb_lm_begin_slots_paged(acb_lm_t* lm, int slots, int max_text, int seq_len_max, int max_prefix, void* k_pool, void* v_pool,
                             int n_pages, int32_t* page_table, int pages_per_row, void* stage_k, void* stage_v,
                             const acb_lm_sampling* sampling, void* stream);

/* acb_lm_begin_slots_paged with an FP8 pool: each K or V vector (64 values of one position, head, layer and row) is 64 e4m3
 * codes (finite variant, max 448) and one fp32 scale, and reads back as code * scale.
 *   k_pool, v_pool    uint8 [L][n_pages][H][ACB_LM_KV_PAGE][64] e4m3 codes
 *   k_scale, v_scale  fp32 [L][n_pages][H][ACB_LM_KV_PAGE]
 * A vector x (the fp32 value the fp16 pool rounds to fp16: after rotary positions for K) is stored as amax = max |x_j|,
 * code_j = cvt.rn.satfinite.e4m3(x_j * (448 / amax)), scale = amax / 448, both divisions correctly rounded; amax == 0
 * stores zero codes and a zero scale.  Decode steps and prompt passes quantize their own K / V; a condition prefix still runs
 * its passes on the fp16 staging cache, whose values admission quantizes into the pages.  Every read of the pool, the
 * position a step has just appended included, sees code * scale.  The cross-attention K/V and the staging cache stay fp16.
 * acb_lm_admit_paged, acb_lm_admit_prompt, acb_lm_steps, acb_lm_step_logits and acb_lm_retire serve the session as they
 * serve an fp16 one.  Everything else is acb_lm_begin_slots_paged. */
int acb_lm_begin_slots_paged_fp8(acb_lm_t* lm, int slots, int max_text, int seq_len_max, int max_prefix, void* k_pool,
                                 void* v_pool, float* k_scale, float* v_scale, int n_pages, int32_t* page_table,
                                 int pages_per_row, void* stage_k, void* stage_v, const acb_lm_sampling* sampling, void* stream);

/* acb_lm_admit_prefix in a paged session: pages [2][n / 2] (host memory) are the page ids of the slot's cond row (slot) and
 * null row (slots + slot), n = 2 * ceil((prefix_len + seq_len) / ACB_LM_KV_PAGE).  The caller gives pages no other live slot
 * holds.  Returns ACB_ERR_INVALID before enqueuing anything when n is not that count, an id is outside [0, n_pages), an id
 * appears twice, or prefix_len > max_prefix; else what acb_lm_admit_prefix checks.  The prefix K/V in the pages are, bit for
 * bit, what acb_lm_admit_prefix writes into a contiguous session's rows.  acb_lm_admit and acb_lm_admit_prefix return
 * ACB_ERR_INVALID in a paged session. */
int acb_lm_admit_paged(acb_lm_t* lm, int slot, const float* cross, int text_len, const float* prefix, int prefix_len,
                       int seq_len, uint64_t seed, const acb_lm_sampling* sampling, const int32_t* pages, int n, void* stream);

/* acb_lm_admit_prefix (pages == NULL, contiguous session) or acb_lm_admit_paged (pages, n_page_ids) that also prefills the
 * request's prompt: after the prefix, sequence columns [0, prefill_cols) of buffers.seq[slot] (their tokens written by the
 * caller) fill cache positions prefix_len + column of the slot's two rows, in the passes acb_lm_prefill runs for a generation
 * of batch 1 with CFG (ACB_LM_PREFILL_ROWS / 2 positions per pass, ACB_LM_PREFILL_PER honoured), so the K/V are bit for bit
 * the ones that generation writes.  The slot then starts at column prefill_cols (acb_lm_slot_status reports it) and finishes
 * after seq_len - 1 - prefill_cols steps.  In a paged session the passes write and read the slot's pages through the page
 * table; nothing is staged for the prompt.  Needs 0 <= prefill_cols <= seq_len - 2 (else ACB_ERR_INVALID, before anything is
 * enqueued) and whatever the call without a prompt needs.  prefill_cols == 0 is acb_lm_admit_prefix / acb_lm_admit_paged. */
int acb_lm_admit_prompt(acb_lm_t* lm, int slot, const float* cross, int text_len, const float* prefix, int prefix_len,
                        int seq_len, int prefill_cols, uint64_t seed, const acb_lm_sampling* sampling, const int32_t* pages,
                        int n_page_ids, void* stream);

/* Cancel the request in `slot` between steps: an ACTIVE or FINISHED slot becomes INACTIVE (status 0) and the next step skips
 * it, as it skips a slot never admitted; the slot is free for acb_lm_admit, which overwrites its K/V, mask and state.  One
 * single-thread kernel on the stream; retiring an INACTIVE slot changes nothing. */
int acb_lm_retire(acb_lm_t* lm, int slot, void* stream);

/* out [slots][2] int32 (device): each slot's position (columns consumed) and status (0 never admitted, 1 decoding,
 * 2 finished). */
int acb_lm_slot_status(acb_lm_t* lm, int* out, void* stream);

/* Teacher-forced / inspection variant of one step: same as acb_lm_steps(1) and additionally leaves the
 * CFG-mixed logits [batch][n_q][card] fp32 in logits_out (may be NULL; in slot mode [slots][n_q][card], active slots only). */
int acb_lm_step_logits(acb_lm_t* lm, float* logits_out, void* stream);

/* Measurement hook: enqueue ONLY the weight-streaming GEMMs (lm_gemm_kernel, lm_gemm_wide_kernel above 64 rows) of one decode step, all layers in step
 * order, so bench.py can time the dominant kernel with CUDA events in isolation.  *n_launches = kernels enqueued. */
int acb_lm_debug_gemms(acb_lm_t* lm, void* stream, int* n_launches);

/* Always 0: the captured decode step chains its kernels with plain stream-order edges, not programmatic dependent launch. */
int acb_lm_uses_pdl(const acb_lm_t* lm);

/* rows the activation buffers must be padded to for `rows` live rows: 16, 32 or 64 up to 64 rows, 128 for 65-128 and 256 for
 * 129-256 (the wide GEMM's tile heights); ACB_ERR_INVALID above ACB_LM_MAX_ROWS. */
int acb_lm_rows_pad(int rows);

/* Number of kernel launches one decode step enqueues (bench.py reports gpu_launches from it). */
int acb_lm_launches_per_step(const acb_lm_t* lm);

/* ---------------------------------------------------------------- MusicGen: LM full-sequence forward -- */

/* LMModel.forward on whole sequences (audiocraft/models/lm.py:221-268; the computation under compute_predictions,
 * lm.py:270-321): causal self attention over every position, no KV cache and no acb_lm_t.  Stateless: it neither reads nor
 * writes any decode handle.
 *   seq     [batch][n_q][seq_len] int64 tokens.  Precondition (not checked on the device, which would break graph capture):
 *           every token lies in [0, card] (card = the special token).
 *   cross   [batch][text_len][d] fp32 condition tensor (cross_attention_src; padded positions are zeros and are attended to,
 *           as in the reference), required exactly when cfg->cross_attention; no CFG rows are added.
 *   prefix  [batch][prefix_len][d] fp32 condition prefix of a `prepend` fuser (MusicGen-melody) or NULL with prefix_len 0: it
 *           runs as the first prefix_len positions (each value rounded to fp16 first) and its logits are not written.
 *   logits  [batch][n_q][seq_len][card] fp32 (the reference returns fp16 under CUDA autocast).
 *   workspace: at least acb_lm_forward_workspace_bytes(...) bytes of device memory, 256-byte aligned.
 * cfg->max_rows, max_seq and max_text are ignored.  Needs dim = 64 * num_heads <= 2048, ffn_dim % 8 == 0, even card,
 * n_q <= 16.  Every output element is summed in one fixed order (no split-K): an item's logits are bit-identical whatever
 * batch it is in.  Tensor maps are encoded per call; all work is on `stream`.  With cfg->weight_dtype 1 a kernel writes each
 * layer's seven matrices as fp16(code * scale) into the workspace before that layer's GEMMs, which read them from there: the
 * workspace is larger by one layer's matrices (fp16). */
int64_t acb_lm_forward_workspace_bytes(const acb_lm_config* cfg, int batch, int prefix_len, int seq_len, int text_len);
int acb_lm_forward(const acb_lm_config* cfg, const acb_lm_weights* w, const int64_t* seq, const float* cross,
                   const float* prefix, int batch, int prefix_len, int seq_len, int text_len, float* logits,
                   void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------- T5 text encoder ------------------ */

/* The text conditioner of MusicGen / AudioGen (T5Conditioner, audiocraft/modules/conditioners.py:422-515): transformers'
 * T5EncoderModel forward (a frozen t5-small / base / large) followed by output_proj and the mask:
 *   out = (output_proj(T5(ids, mask)) * mask) */
typedef struct {
    int d_model;      /* multiple of 64, <= 2048 */
    int d_kv;         /* must be 64 (t5-3b / t5-11b use 128: refused) */
    int num_heads;    /* num_heads * d_kv == d_model */
    int num_layers;
    int d_ff;         /* multiple of 4; the feed-forward is wo(relu(wi(x))) */
    int vocab_size;
    int num_buckets;  /* relative_attention_num_buckets */
    int out_dim;      /* output_proj out_features, multiple of 4 */
    float eps;        /* layer_norm_epsilon */
} acb_t5_config;

/* fp32 matrices in the [out_features][in_features] layout of transformers' T5, stacked over layers; no biases but proj_b. */
typedef struct {
    const float* shared;   /* [vocab][d]          shared.weight */
    const float* w_qkv;    /* [L][3d][d]          layer.0.SelfAttention.{q,k,v}.weight, stacked q, k, v */
    const float* w_o;      /* [L][d][d]           layer.0.SelfAttention.o.weight */
    const float* w_i;      /* [L][d_ff][d]        layer.1.DenseReluDense.wi.weight */
    const float* w_fo;     /* [L][d][d_ff]        layer.1.DenseReluDense.wo.weight */
    const float* ln;       /* [L][2][d]           layer.0.layer_norm.weight, layer.1.layer_norm.weight */
    const float* final_ln; /* [d]                 encoder.final_layer_norm.weight */
    const float* rel_bias; /* [num_buckets][H]    block.0 ... relative_attention_bias.weight, used by every layer */
    const float* proj_w;   /* [out_dim][d]        the conditioner's output_proj.weight */
    const float* proj_b;   /* [out_dim]           output_proj.bias */
} acb_t5_weights;

/* ids     [batch][seq_len] int64 token ids.  Precondition (not checked on the device): every id lies in [0, vocab_size).
 * mask    [batch][seq_len] int64 attention mask (0 or 1).  Keys with mask 0 are not attended to; output rows with mask 0 are
 *         exact zeros.  A row whose mask is all zero therefore comes out as exact zeros (its queries attend to nothing).
 * buckets [2 seq_len - 1] int32: buckets[j - i + seq_len - 1] is the bidirectional relative-position bucket of key j seen from
 *         query i (T5Attention._relative_position_bucket; audiocraft_b200.t5.relative_position_buckets computes it).
 * out     [batch][seq_len][out_dim] fp32.
 * hidden  [batch][seq_len][d] fp32 T5 last_hidden_state, or NULL.
 * workspace: at least acb_t5_workspace_bytes(...) bytes of device memory, 256-byte aligned.
 * GEMMs on the TF32 tensor pipe (fp32 operands, fp32 accumulation), q / k / v rounded to fp16 for the attention products,
 * softmax and everything else fp32.  No split-K: an item's outputs are bit-identical whatever batch it is in and however
 * far past its length the batch is padded.  Stateless, graph-capturable; all work is on `stream`. */
int64_t acb_t5_workspace_bytes(const acb_t5_config* cfg, int batch, int seq_len);
int acb_t5_encode(const acb_t5_config* cfg, const acb_t5_weights* w, const int64_t* ids, const int64_t* mask,
                  const int32_t* buckets, int batch, int seq_len, float* out, float* hidden, void* workspace,
                  int64_t workspace_bytes, void* stream);

/* Stand-alone sampler (tail of _sample_next_token, lm.py:403-418; utils/utils.py:88-141) for unit tests:
 * logits [rows][n_q][card] fp32 ([cond; null] rows when rows == 2*batch), noise optional, tokens [batch][n_q]. */
int acb_sample(const float* logits, const float* noise, int64_t* tokens, int batch, int rows, int n_q, int card,
               const acb_lm_sampling* sampling, uint64_t step, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AUDIOCRAFT_B200_H */
