"""Full-sequence forward (LMModel.compute_predictions on acb_lm_forward) against the decode path and a torch eager fp16
forward on the same weights: CUDA-event times after warm-up, algorithmic TFLOP/s from the shapes and their share of the
H100's 989 TFLOP/s dense fp16 peak, the GEMM / attention / other split of the forward from a torch.profiler run, and the
max |logit difference| to the eager forward.  Prints the GPU name and power limit.
    python profiles/perf_forward.py [--only medium]"""
import argparse
import math
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200.loaders import load_lm_model  # noqa: E402

PEAK = 989e12
WORKLOADS = [('medium', 8, 1500), ('large', 8, 1500), ('small', 32, 500)]
TEXT = 16


def gpu_name():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def flops(lm, B, S, Tt):
    d, ffn, L = lm.dim, lm.ffn_dim, lm.num_layers
    tok = B * S
    mm = tok * L * 2 * (4 * d * d + 2 * d * ffn + (2 * d * d if lm.cross_attention else 0)) + tok * 2 * d * lm.n_q * lm.card
    mm += (B * Tt * L * 2 * 2 * d * d) if lm.cross_attention else 0
    att = B * L * 4 * d * S * (S + 1) / 2 + ((B * L * 4 * d * S * Tt) if lm.cross_attention else 0)
    return mm, att


@torch.no_grad()
def eager_forward(lm, seq, cross):
    """The reference's arithmetic under CUDA autocast, in plain torch: fp16 GEMMs (F.linear) and SDPA, fp32 LayerNorm and
    residual stream."""
    w, d, H = lm._w, lm.dim, lm.num_heads
    B, K, S = seq.shape
    x = sum(F.embedding(seq[:, k], w['emb'][k]).float() for k in range(K))
    pos = torch.arange(S, device=seq.device, dtype=torch.float32).view(1, -1, 1)
    x = x + float(lm.cfg_dict.get('positional_scale', 1.0)) * torch.cat([torch.cos(pos / w['inv_freq']), torch.sin(pos / w['inv_freq'])], -1)
    c16 = cross.half() if cross is not None else None

    def heads(t):
        return t.view(B, -1, H, 64).transpose(1, 2)

    def ln(v, wb):
        return F.layer_norm(v, (d,), wb[0], wb[1], 1e-5).half()
    for li in range(lm.num_layers):
        lw = w['ln'][li]
        q, k, v = F.linear(ln(x, lw[0:2]), w['w_qkv'][li]).split(d, dim=-1)
        a = F.scaled_dot_product_attention(heads(q), heads(k), heads(v), is_causal=True)
        x = x + F.linear(a.transpose(1, 2).reshape(B, S, d), w['w_o'][li]).float()
        if c16 is not None:
            q = F.linear(ln(x, lw[2:4]), w['w_cq'][li])
            k, v = F.linear(c16, w['w_ckv'][li]).split(d, dim=-1)
            a = F.scaled_dot_product_attention(heads(q), heads(k), heads(v))
            x = x + F.linear(a.transpose(1, 2).reshape(B, S, d), w['w_co'][li]).float()
        x = x + F.linear(F.gelu(F.linear(ln(x, lw[4:6]), w['w_ff1'][li])), w['w_ff2'][li]).float()
    h = ln(x, w['out_norm'])
    return F.linear(h, w['heads']).float().view(B, S, K, lm.card).permute(0, 2, 1, 3)


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = math.inf
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best


def split(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    t = {'gemm': 0.0, 'attention': 0.0, 'other': 0.0}
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
        key = 'gemm' if 'lm_fwd_gemm' in ev.key else ('attention' if 'lm_fwd_attn' in ev.key else 'other')
        t[key] += us / 1e3
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--only', default=None)
    a = ap.parse_args()
    print('GPU:', gpu_name())
    for scale, B, T in WORKLOADS:
        if a.only and scale != a.only:
            continue
        lm = load_lm_model(f'synthetic/{scale}')
        g = torch.Generator(device='cuda').manual_seed(1)
        codes = torch.randint(0, lm.card, (B, lm.n_q, T), device='cuda', generator=g)
        cross = torch.randn(B, TEXT, lm.dim, device='cuda', generator=g) * 0.1
        seq = lm.pattern_provider.get_pattern(T).build_pattern_sequence(codes, lm.card, keep_only_valid_steps=True)[0]
        S = seq.shape[-1]
        mm, att = flops(lm, B, S, TEXT)
        t_fwd = timed(lambda: lm.compute_predictions(codes, cross_attention_src=cross))
        t_eager = timed(lambda: eager_forward(lm, seq, cross))
        sp = split(lambda: lm.forward(seq, cross_attention_src=cross))
        diff = float((lm.forward(seq, cross_attention_src=cross) - eager_forward(lm, seq, cross)).abs().max())
        # decode path: one warm-up pass (buffer allocation, graph capture) before the timed one; a pass is S - 1 steps
        t_dec = timed(lambda: lm.teacher_forced_logits(seq, cross, 1.0, n_steps=S - 1, keep=[S - 2]), reps=1)
        tf = (mm + att) / (t_fwd * 1e-3) / 1e12
        gemm_tf = mm / (sp['gemm'] * 1e-3) / 1e12 if sp['gemm'] else float('nan')
        print(f'{scale} B={B} T={T} (S={S}, {B * S} tokens, {(mm + att) / 1e12:.1f} TFLOP: {mm / 1e12:.1f} GEMM + {att / 1e12:.2f} attention)')
        print(f'  compute_predictions {t_fwd:8.1f} ms  {tf:6.1f} TFLOP/s = {tf * 1e12 / PEAK * 100:.1f} % of 989')
        print(f'  split (profiler)    gemm {sp["gemm"]:.1f} ms ({gemm_tf:.0f} TFLOP/s, {gemm_tf * 1e12 / PEAK * 100:.0f} %), '
              f'attention {sp["attention"]:.1f} ms, other {sp["other"]:.1f} ms')
        print(f'  torch eager fp16    {t_eager:8.1f} ms  ({t_eager / t_fwd:.2f}x the forward); max |logit diff| {diff:.4f}')
        print(f'  decode path         {t_dec:8.1f} ms  ({S - 1} teacher-forced steps; {t_dec / t_fwd:.0f}x the forward)')
        del lm
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
