// Internal interface between lm.cu (handle, graph capture, sampler) and lm_step.cu (the persistent fused decode step).
#pragma once
#include "common.cuh"

constexpr int ACB_STEP_GEMMS = 7;          // QKV, O, CQ, CO, FF1, FF2, HEADS
enum { SG_QKV = 0, SG_O = 1, SG_CQ = 2, SG_CO = 3, SG_FF1 = 4, SG_FF2 = 5, SG_HEADS = 6 };
constexpr int ACB_STEP_MAX_SPLIT = 16;     // split-K partial slots in buffers.part
constexpr int ACB_STEP_STAT_CHUNKS = 8;    // LayerNorm statistics are kept per d/8 columns

// How one GEMM of the step is cut into work items: item = (128-feature tile, K slice of kb_per 64-element blocks).
struct StepGemm {
    const __half* wp;      // packed weights (per layer: n_tiles * nkb tiles of 16 KB), see acb_lm_pack_weight
    size_t layer_stride;   // halves between layers (0 for the heads)
    int N, K, n_tiles, nkb, ksplit, kb_per, n_items;
};

struct StepParams {
    int d, H, L, ffn, n_q, card, rows, R, batch, has_cross, text_len, max_seq, max_text, max_rows;
    int n_stage, act_bytes;
    float pos_scale, attn_scale;
    const __half* emb; const float* inv_freq; const float* ln; const float* out_norm;
    StepGemm g[ACB_STEP_GEMMS];
    float* x; float* part; float* stats; __half* a16; __half* h16; float* logits;
    __half* kc; __half* vc; const __half* ckc; const __half* cvc;
    const int64_t* seq; const int* pos; unsigned* bar;
    unsigned long long* trace;   // debug: CTA 0 stamps %globaltimer after every grid barrier (NULL: off)
    int l2_ahead;                // tiles the producer's L2-prefetch cursor runs ahead of its ring cursor
    int stop_after, max_gemms;   // debug (ACB_LM_STEP_STOP): leave the kernel after this many grid barriers
    int sin_pos, rope;           // positional_embedding: 'sin' (1,0), 'rope' (0,1), 'sin_rope' (1,1)  (transformer.py:632-637, 701-705)
    const float* rope_freq;      // [32] 1 / max_period^(2i/64), RotaryEmbedding.frequencies (rope.py:68-69)
};

struct StepLaunch {
    StepParams p;
    int grid, block;
    size_t smem;
    int n_phases;          // grid barriers per step + 1
    bool cooperative;
};

// Fills `out` for the current (rows, cross) configuration; returns ACB_ERR_INVALID (with acb_last_error) when the
// shapes are not supported by the fused step.
int lm_step_prepare(const acb_lm_config& cfg, const acb_lm_weights& w, const acb_lm_buffers& b, int rows, int batch,
                    int text_len, bool has_cross, int sms, StepLaunch* out);
int lm_step_launch(const StepLaunch& L, cudaStream_t s);
