"""The decode step's non-GEMM kernels against float64, computed from each kernel's own inputs read back from the buffers the
caller owns, at per-slot positions, text lengths and page boundaries.

tests/test_gpu_kernels_f64.py checks the forward stages and the decode GEMMs.  The kernels here were otherwise checked end to
end (logits at rtol 2e-2 / atol 3e-2, which absorbs a rotary angle one position off or a causal mask one key off) or against
each other (paged vs contiguous, session vs `generate`), and the slot / paged kernels share their bodies with the contiguous
ones, so a mistake in a shared body passes both.

Probe weights.  Every layer's self / cross out-projection and linear2 are zero and every norm is a copy of out_norm, so the
residual stream stays the embedding and, after a step or a pass, `h16` is bit for bit the input of every layer's QKV, cross-q
and FF1 GEMM.  With cross attention W_cq (the first d rows of the cross in-projection) is the identity: each cross-query sum
has one non-zero product, the `part` slots add up to exactly h16, and the cross kernel's query is h16.  After a step `q32`
holds the last layer's self-attention query, `a16` the self-attention output (no cross attention) or the cross-attention
output (cross attention), and the caches every layer's K / V.  Before each checked step every cache position the step must not
read is NaN (positions >= n - 1 of active rows, every row of a slot not decoding, every free page and the unwritten offsets
of a row's pages, cross positions >= the slot's own text length): the kernels guard every load with `pp < n` / `t < n`, so a
NaN read shows in the output.  The step must change exactly position n - 1 of each active row in every layer.

Bounds.  Embedding: (n_q - 1) 2^-24 sum_k |e_k| for the fp32 sum of the fp16 rows, 2 2^-24 |x| for the rounding of the sin term
and the final add, and 2^-21 pos_scale for cosf / sinf (<= 2 ulp of a value <= 1) of the fp32 phase pos / inv_freq[j], which the
reference forms in fp32 as the kernel does.  LayerNorm: check_ln.  Rotary positions: check_rope at each row's own position.
Cross K/V: check_gemm_f16.  The residual fold of lm_ln_kernel is compared bit for bit.

Attention (attn_decode64).  With w_i the float64 softmax weights, o the float64 output and s_i the scores q.k_i / 8:
  * scores: an fp32 FMA chain of 8 products and a 3-level shuffle tree (the self kernels) or a 64-product chain (cross); every
    partial sum is <= S_i = sum_j |q_j k_ij| / 8, so |s~_i - s_i| <= delta_i = 64 2^-24 S_i (any order of 64 terms).  A score
    error e_i moves the output by sum_i w_i (v_i - o) e_i to first order (the common part of e cancels in the normalisation);
    2 delta_i covers the second order.
  * weights: __expf is ex2.approx (relative error < 2^-22) of x log2(e) rounded to fp32 (relative 2^-24 |x|): per call
    2^-21 + 2^-24 |s_i - m|.  A key's weight passes through its own __expf and at most one rescale per iteration of its lane,
    plus the 2 group merges, the warp merge and the final division: eps = (n_it + 4)(2^-21 + 2^-24 max_i |s_i - m|), n_it =
    ceil(n / 32) the lane's iterations (the cross kernel's chunks of 32).  A relative weight error moves the output by at most
    sum_i w_i |v_i - o| eps.
  * accumulation: fp32, each accumulator a chain of the keys of one lane (ceil(n / 32) in the self kernels, all n in the cross
    kernel, whose lanes hold output dims), each step one rounding of at most 2^-24 of the running |sum|, plus 16 for the
    merges, the normaliser and the division: (acc + 16) 2^-24 sum_i w_i |v_i|.
  * output: half an fp16 ulp.
The CPU self-check shows the bound is sharp: an fp32 emulation of the self kernel's partition (8 warps x 4 position groups,
online softmax, group and warp merges) passes at n = 1503, while a missing newest or oldest key, one extra key, a full page
swapped with the row's last page, swapped heads or another slot's n fail.  (2^-10 max|v|, the forward kernels' bound, is
larger than the effect of one key, |v| / n, from n ~ 1000 on.)

Measured on an H100 80GB HBM3 at a 700 W limit (the file's GPU tests take about 30 s): the worst element of the attention
checks reached 0.99 of the bound at short key counts, where half an fp16 ulp of the output dominates, and 0.94 at n = 1503;
cross attention 0.96; K / V in the caches 0.998 and LayerNorm 1.0 (both one fp16 rounding); q32 0.99; the embedding 0.24.

Coverage: each kernel of csrc/lm.cu the decode step, its prefill passes and admission launch, and the test that checks it.
  lm_embed_kernel<false>              test_generate_step_matches_float64 (every case)
  lm_embed_kernel<true>               test_prefill_passes_match_float64[contiguous-*] (acb_lm_prefill), [paged-*] (admission)
  lm_embed_slot_kernel                test_slot_step_matches_float64 (every case; sin term at prefix + column: melody-*)
  lm_embed_prefix_kernel              test_prefill_passes_match_float64[melody-*]
  lm_ln_kernel                        every test; d = 128 (tiny), 256 (mini), 1536 (medium), 2048 (large); the residual fold
                                      bit for bit: test_generate_step_matches_float64[mini-sin-B6], [tiny-sin-B32]
  lm_qkv_slot_kernel                  test_slot_step_matches_float64[*-contiguous]; prefixes 9, 63, 64, 65, 0 side by side:
                                      [melody-sin-5-contiguous]
  lm_qkv_slot_paged_kernel            test_slot_step_matches_float64[*-paged]; with prefixes: [melody-sin_rope-5-paged]
  lm_qkv_pf_paged_kernel              test_prefill_passes_match_float64[paged-*]
  lm_gemm_kernel<*, EPI_QKV(_ROPE)>   K/V / q32 at the step's position: test_generate_step_matches_float64
  lm_gemm_kernel<*, EPI_QKV_PF*>      test_prefill_passes_match_float64[contiguous-*], [melody-*]
  lm_gemm_kernel<8, EPI_CROSSKV>      at acb_lm_begin: test_generate_step_matches_float64 (cross cases); at admission:
                                      test_slot_step_matches_float64 (cross cases; T = 65 and 129 leave a 1-row last
                                      chunk of admission's 64-row loop, 150 a 22-row one)
  lm_attn2_kernel<false>              test_generate_step_matches_float64 (no cross attention), n up to 1503
  lm_attn2_kernel<true>               test_prefill_passes_match_float64[contiguous-rope-B1], [melody-*]; the cross cases
                                      [contiguous-*-cross] run it too, but their a16 holds the cross-attention output, so
                                      there it is covered only by the NaN caches and the K / V it leaves behind
  lm_attn2_slot_kernel                test_slot_step_matches_float64[*-nocross-*-contiguous], [melody-sin-5-contiguous]
  lm_attn2_slot_paged_kernel          test_slot_step_matches_float64[*-nocross-*-paged], [melody-sin_rope-5-paged]
  lm_attn2_pf_paged_kernel            test_prefill_passes_match_float64[paged-*]
  lm_cross_attn_kernel<false>         test_generate_step_matches_float64 (cross cases, double CFG included)
  lm_cross_attn_kernel<true>          test_prefill_passes_match_float64[contiguous-*-cross]
  lm_cross_attn_slot_kernel           test_slot_step_matches_float64[*-cross-*]
Not here: the decode GEMMs and forward stages (tests/test_gpu_kernels_f64.py); lm_sample_kernel / lm_sample_slot_kernel
(tests/test_gpu_lm.py against the oracle); lm_prefix_scatter_kernel (tests/test_gpu_continuous_paged.py, bit for bit against
the staging cache); the bookkeeping kernels lm_slot_sampling_kernel, lm_slot_admit_kernel, lm_slot_retire_kernel,
lm_page_table_kernel, lm_set_pos_kernel and lm_f32_to_f16_kernel (through every session and generation test of
tests/test_gpu_continuous*.py).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from audiocraft_b200 import _lib
from oracle import lm_oracle as LO
from tests.test_gpu_edges import _swap
from tests.test_gpu_kernels_f64 import U, _nt_rows_pad, _synth, check, check_gemm_f16, check_ln, check_rope, gemm64, half_ulp16, \
    probe_state_dict

PAGE = _lib.ACB_LM_KV_PAGE
NAN = float('nan')


# ----------------------------------------------------------------------------- float64 references and bounds

def attn_decode64(q, k, v, acc, n_it):
    """float64 softmax(q k^T / 8) v for one query per row and the decode kernels' bound (module docstring).  q [R, H, 64]
    (fp16 values), k / v [R, H, n, 64]; acc: keys per accumulator chain, n_it: iterations (chunks) per lane.  Returns
    (out [R, H * 64], tol)."""
    R, Hn, n, _ = k.shape
    prod = q.double().unsqueeze(2) * k.double() / 8.0                       # [R, H, n, 64]
    s = prod.sum(-1)
    w = torch.softmax(s, -1)
    v64 = v.double()
    o = (w.unsqueeze(-1) * v64).sum(2)                                      # [R, H, 64]
    delta = 64 * U * prod.abs().sum(-1)
    eps = (n_it + 4) * (2.0 ** -21 + U * (s - s.amax(-1, keepdim=True)).abs().amax(-1, keepdim=True))
    t = (w.unsqueeze(-1) * (v64 - o.unsqueeze(2)).abs() * (2 * delta + eps).unsqueeze(-1)).sum(2)
    t = t + (acc + 16) * U * (w.unsqueeze(-1) * v64.abs()).sum(2)
    return o.reshape(R, Hn * 64), (t + half_ulp16(o.abs() + t)).reshape(R, Hn * 64)


def self_attn64(q, k, v):
    n = k.shape[2]
    return attn_decode64(q, k, v, -(-n // 32), -(-n // 32))


def cross_attn64(q, k, v):
    n = k.shape[2]
    return attn_decode64(q, k, v, n, -(-n // 32))


def embed64(w, cfg, toks, pos):
    """x of rows with tokens toks [R, n_q] (clamped as the kernel clamps them) at cache positions pos [R]: sum_k fp16
    emb[k, tok_k] plus pos_scale [cos, sin](fp32(pos / inv_freq)) when the model has the sin term.  Returns (x, tol)."""
    card = cfg['card']
    toks = toks.long().clamp(0, card).where(toks >= 0, torch.full_like(toks, card))
    e = torch.stack([w['emb'][k][toks[:, k].to(w['emb'].device)].double() for k in range(cfg['n_q'])])
    x, tol = e.sum(0), (cfg['n_q'] - 1) * U * e.abs().sum(0)
    return _add_sin(x, tol, w, cfg, pos)


def _add_sin(x, tol, w, cfg, pos):
    if cfg['positional_embedding'] == 'rope':
        return x, tol
    ph = (pos.to(x.device).float().unsqueeze(1) / w['inv_freq'].to(x.device).float().unsqueeze(0)).double()
    x = x + cfg['positional_scale'] * torch.cat([torch.cos(ph), torch.sin(ph)], dim=1)
    return x, tol + 2 * U * x.abs() + 2.0 ** -21 * cfg['positional_scale']


def fold32(x, parts):
    """lm_ln_kernel's residual fold: ((x + p0) + p1) + ... in fp32, slot order."""
    a = x.float().clone()
    for p in parts:
        a = a + p.float()
    return a


def check_fold(got, x, parts, what):
    want = fold32(x, parts)
    bad = int((got != want).sum())
    print(f'{what}: {bad} of {got.numel()} elements differ from the fp32 fold')
    assert bad == 0, f'{what}: the residual fold is not ((x + p0) + p1) + ... bit for bit'


def emulate_self_attn32(q, k, v):
    """fp32 emulation of lm_attn2_kernel's order of operations for one query: keys pp = (k * 8 + warp) * 4 + pg, an online
    softmax per (warp, position group), the groups merged (xor 8, xor 16), then the warps.  q [H, 64], k / v [H, n, 64]."""
    Hn, n, _ = k.shape
    n_it = -(-n // 32)
    pad = n_it * 32 - n
    kp = torch.cat([k.float(), torch.zeros(Hn, pad, 64)], 1).view(Hn, n_it, 8, 4, 64)
    vp = torch.cat([v.float(), torch.zeros(Hn, pad, 64)], 1).view(Hn, n_it, 8, 4, 64)
    live = (torch.arange(n_it * 32) < n).view(n_it, 8, 4)
    qs = q.float() * 0.125
    m = torch.full((Hn, 8, 4), -math.inf)
    l = torch.zeros(Hn, 8, 4)
    acc = torch.zeros(Hn, 8, 4, 64)
    for it in range(n_it):
        part = (qs.view(Hn, 1, 1, 8, 8) * kp[:, it].view(Hn, 8, 4, 8, 8)).sum(-1)       # 8 lanes' chains [H, 8, 4, 8]
        s = ((part[..., 0] + part[..., 1]) + (part[..., 2] + part[..., 3])) + \
            ((part[..., 4] + part[..., 5]) + (part[..., 6] + part[..., 7]))
        mn = torch.maximum(m, s)
        corr, pw = torch.exp(m - mn), torch.exp(s - mn)
        upd = live[it].expand(Hn, 8, 4)
        l = torch.where(upd, l * corr + pw, l)
        acc = torch.where(upd.unsqueeze(-1), acc * corr.unsqueeze(-1) + pw.unsqueeze(-1) * vp[:, it], acc)
        m = torch.where(upd, mn, m)

    def merge(ma, la, aa, mb, lb, ab):
        mn = torch.maximum(ma, mb)
        ca = torch.where(ma == -math.inf, torch.zeros_like(ma), torch.exp(ma - mn))
        cb = torch.where(mb == -math.inf, torch.zeros_like(mb), torch.exp(mb - mn))
        return mn, la * ca + lb * cb, aa * ca.unsqueeze(-1) + ab * cb.unsqueeze(-1)
    m01, l01, a01 = merge(m[..., 0], l[..., 0], acc[..., 0, :], m[..., 1], l[..., 1], acc[..., 1, :])
    m23, l23, a23 = merge(m[..., 2], l[..., 2], acc[..., 2, :], m[..., 3], l[..., 3], acc[..., 3, :])
    mw, lw, aw = merge(m01, l01, a01, m23, l23, a23)                                     # [H, 8]
    mx = mw.amax(-1, keepdim=True)
    cw = torch.where(mw == -math.inf, torch.zeros_like(mw), torch.exp(mw - mx))
    lt, ot = torch.zeros(Hn), torch.zeros(Hn, 64)
    for wi in range(8):
        lt = lt + lw[:, wi] * cw[:, wi]
        ot = ot + aw[:, wi] * cw[:, wi].unsqueeze(-1)
    return (ot / lt.unsqueeze(-1)).half().reshape(Hn * 64)


def emulate_cross_attn32(q, k, v):
    """fp32 emulation of cross_attn_body: chunks of 32 text positions, a sequential 64-product score chain per lane."""
    Hn, n, _ = k.shape
    qs = q.float() * 0.125
    mx, l, o = torch.full((Hn,), -math.inf), torch.zeros(Hn), torch.zeros(Hn, 64)
    for t0 in range(0, n, 32):
        s = (qs.unsqueeze(1) * k[:, t0:t0 + 32].float()).sum(-1)                         # [H, <=32]
        cm = torch.maximum(mx, s.amax(-1))
        corr = torch.where(mx == -math.inf, torch.zeros_like(mx), torch.exp(mx - cm))
        pw = torch.exp(s - cm.unsqueeze(-1))
        l = l * corr + pw.sum(-1)
        o = o * corr.unsqueeze(-1)
        for j in range(s.shape[1]):
            o = o + pw[:, j:j + 1] * v[:, t0 + j].float()
        mx = cm
    return (o / l.unsqueeze(-1)).half().reshape(Hn * 64)


# ----------------------------------------------------------------------------- CPU self-check

def test_decode_float64_checks_accept_kernel_arithmetic_and_reject_mutations():
    """CPU: each check accepts an fp32 / fp16 emulation of its kernel's arithmetic and rejects: for self attention at n = 1503
    a missing newest or oldest key, one extra key, a full page swapped with the row's last page, swapped heads and another
    slot's n; for cross attention another slot's text length; for rotary positions another slot's position; for the
    embedding the position one off either way; for the residual fold one part slot left out and the reversed order."""
    g = torch.Generator().manual_seed(3)
    Hn, n = 4, 1503
    q = torch.randn(1, Hn, 64, generator=g).half()
    k = torch.randn(1, Hn, n + 1, 64, generator=g).half()
    v = torch.randn(1, Hn, n + 1, 64, generator=g).half()
    kern = emulate_self_attn32(q[0], k[0, :, :n], v[0, :, :n]).unsqueeze(0)
    ref, tol = self_attn64(q, k[:, :, :n], v[:, :, :n])
    check(kern, ref, tol, 'self-check self attention n=1503')
    for nn in (1, 2, 31, 33, 65, 257):
        r, t = self_attn64(q, k[:, :, :nn], v[:, :, :nn])
        check(emulate_self_attn32(q[0], k[0, :, :nn], v[0, :, :nn]).unsqueeze(0), r, t, f'self-check self attention n={nn}')
    # the page table of a row: pages 0 .. 23, position p at offset p % 64 of page p // 64; the last page is partial
    last = (n - 1) // PAGE
    perm = torch.arange(n)
    first = torch.arange(PAGE)
    perm_sw = torch.cat([last * PAGE + first, perm[PAGE:last * PAGE], first[:n - last * PAGE]])
    kv_pool_k = torch.cat([k[:, :, :n], torch.randn(1, Hn, (last + 1) * PAGE - n, 64, generator=g).half()], 2)
    kv_pool_v = torch.cat([v[:, :, :n], torch.randn(1, Hn, (last + 1) * PAGE - n, 64, generator=g).half()], 2)
    mutants = {
        'newest key dropped': (k[:, :, :n - 1], v[:, :, :n - 1]),
        'oldest key dropped': (k[:, :, 1:n], v[:, :, 1:n]),
        'one extra key': (k, v),
        'page 0 swapped with the last page': (kv_pool_k[:, :, perm_sw], kv_pool_v[:, :, perm_sw]),
        "another slot's n (n - 5)": (k[:, :, :n - 5], v[:, :, :n - 5]),
    }
    for what, (kk, vv) in mutants.items():
        with pytest.raises(AssertionError):
            check(emulate_self_attn32(q[0], kk[0], vv[0]).unsqueeze(0), ref, tol, what)
    with pytest.raises(AssertionError):
        check(_swap(kern.view(1, Hn, 64), 0, dim=1).reshape(1, Hn * 64), ref, tol, 'swapped heads')

    # cross attention: text lengths on both sides of the 32-position chunks
    ck = torch.randn(1, Hn, 150, 64, generator=g).half()
    cv = torch.randn(1, Hn, 150, 64, generator=g).half()
    for T, T_other in ((1, 31), (32, 33), (65, 64), (150, 65)):
        r, t = cross_attn64(q, ck[:, :, :T], cv[:, :, :T])
        check(emulate_cross_attn32(q[0], ck[0, :, :T], cv[0, :, :T]).unsqueeze(0), r, t, f'self-check cross T={T}')
        with pytest.raises(AssertionError):
            check(emulate_cross_attn32(q[0], ck[0, :, :T_other], cv[0, :, :T_other]).unsqueeze(0), r, t,
                  f"cross T={T} with the other slot's T={T_other}")

    # rotary positions, one row per slot at its own position
    cfg = dict(max_period=10000.0, positional_scale=1.0)
    R = 4
    a = torch.randn(R, 256, generator=g).half()
    wq = (torch.randn(Hn * 64, 256, generator=g) / 16).half()
    v64, bnd = gemm64(a, wq)
    v64, bnd = v64.view(R, Hn, 1, 64), bnd.view(R, Hn, 1, 64)
    pos = torch.tensor([1502, 1501, 64, 0])
    f32 = (a.float() @ wq.float().t()).view(R, Hn, 1, 64).half().float()
    kern = torch.cat([LO.rope_rotate(f32[i:i + 1], int(p), 1e4, 1.0) for i, p in enumerate(pos.tolist())])
    check_rope(kern, v64, bnd, pos, cfg, False, 'self-check rope per row')
    check_rope(kern.half(), v64, bnd, pos, cfg, True, 'self-check rope per row fp16')
    with pytest.raises(AssertionError):
        check_rope(kern, v64, bnd, pos[[1, 0, 3, 2]], cfg, False, "rope at the neighbouring slot's position")

    # embedding at per-row positions
    ecfg = dict(card=64, n_q=4, positional_embedding='sin', positional_scale=1.0)
    d = 128
    adim = torch.arange(d // 2, dtype=torch.float32)
    w = dict(emb=(torch.randn(4, 65, d, generator=g) * 0.5).half(), inv_freq=torch.tensor(1e4) ** (adim / (d // 2 - 1)))
    toks = torch.randint(-1, 66, (R, 4), generator=g)
    pos = torch.tensor([1502, 257, 64, 0])
    tk = toks.clamp(0, 64).where(toks >= 0, torch.full_like(toks, 64))
    x32 = torch.zeros(R, d)
    for kq in range(4):
        x32 = x32 + w['emb'][kq][tk[:, kq]].float()
    ph = pos.float().unsqueeze(1) / w['inv_freq'].unsqueeze(0)
    x32 = x32 + torch.cat([torch.cos(ph), torch.sin(ph)], 1)
    ref, tol = embed64(w, ecfg, toks, pos)
    check(x32, ref, tol, 'self-check embedding')
    for dp in (-1, 1):
        r2, t2 = embed64(w, ecfg, toks, pos + dp)
        with pytest.raises(AssertionError):
            check(x32[:3], r2[:3], t2[:3], f'embedding at position {dp:+d}')

    # LayerNorm at the widths of the released models, and the residual fold
    for dd in (128, 256, 1536, 2048):
        x = torch.randn(3, dd, generator=g) * 2 + 0.5
        gm, bt = 1 + 0.1 * torch.randn(dd, generator=g), 0.05 * torch.randn(dd, generator=g)
        check_ln(F.layer_norm(x, (dd,), gm, bt, 1e-5).half(), x, gm, bt, f'self-check LayerNorm d={dd}')
    x = torch.randn(8, 256, generator=g) * 3
    parts = [torch.randn(8, 256, generator=g) * 10.0 ** (-(i % 4)) for i in range(_lib.ACB_LM_MAX_SPLIT)]
    got = fold32(x, parts)
    check_fold(got, x, parts, 'self-check fold')
    with pytest.raises(AssertionError):
        check_fold(got, x, parts[:3] + parts[4:], 'fold without part slot 3')
    with pytest.raises(AssertionError):
        check_fold(got, x, parts[::-1], 'fold in reverse order')


# ----------------------------------------------------------------------------- GPU helpers

def _probe(name, pe, cross, prefix=False, seed=7):
    """The probe LM (module docstring) on `name`'s synthetic weights; returns (cfg, original state dict, LMModel)."""
    from audiocraft_b200.conditioners import ConditionFuser
    from audiocraft_b200.lm import LMModel
    cfg0, sd0 = _synth(name, (), cross, seed)
    cfg = dict(cfg0, positional_embedding=pe)
    sd = probe_state_dict(cfg, sd0, ('self_attn.out_proj.weight', 'cross_attention.out_proj.weight', 'linear2.weight'), True)
    if cross:
        d = cfg['dim']
        for li in range(cfg['num_layers']):
            p = f'transformer.layers.{li}.cross_attention.in_proj_weight'
            sd[p] = sd[p].clone()
            sd[p][:d] = torch.eye(d)
    fuser = ConditionFuser({'prepend': ['self_wav', 'description']}) if prefix else None
    return cfg, sd0, LMModel(sd, cfg, None, fuser)


def _heads(t, R, Hn):
    return t.reshape(R, Hn, 1, 64)


def _nan_equal(a, b):
    return (a == b) | (torch.isnan(a) & torch.isnan(b))


def check_qkv(m, cfg, h, pos, kv_at, tag, q32=None):
    """q32 rows (last layer) and every layer's K / V at each row's own cache position pos [R]: kv_at(layer, 'k' | 'v') ->
    [R, H, 64] read back at those positions."""
    w, d, Hn, NL = m._w, cfg['dim'], cfg['num_heads'], cfg['num_layers']
    R, rope = h.shape[0], cfg['positional_embedding'] != 'sin'
    for layer in range(NL):
        v64, bnd = gemm64(h, w['w_qkv'][layer])
        for i, n in enumerate(('q', 'k', 'v')):
            if n == 'q' and (layer != NL - 1 or q32 is None):
                continue
            got = q32.reshape(R, Hn, 1, 64) if n == 'q' else kv_at(layer, n).reshape(R, Hn, 1, 64)
            r, e = _heads(v64[:, i * d:(i + 1) * d], R, Hn), _heads(bnd[:, i * d:(i + 1) * d], R, Hn)
            what = f'{tag} layer {layer} {n}'
            if rope and n != 'v':
                check_rope(got, r, e, pos.cpu(), cfg, n != 'q', what + ' (rope)')
            elif n == 'q':
                check(got, r, e, what)
            else:
                check_gemm_f16(got, r, e, what)


def check_attention(a16, q, groups, tag, cross=False):
    """a16 rows against attention over their own keys: groups = [(row indices, k [R, H, n, 64], v)]."""
    for rows, k, v in groups:
        ref, tol = (cross_attn64 if cross else self_attn64)(q[rows], k, v)
        check(a16[rows], ref, tol, f'{tag} {"cross" if cross else "self"} attention n={k.shape[2]} rows {rows.tolist()[:4]}..')


# ----------------------------------------------------------------------------- continuous-batching step

# (id, model, positional embedding, cross attention, slots, paged, max_gen_len, checkpoints (steps of slot 0))
CHECKPOINTS = (0, 1, 30, 31, 32, 62, 63, 64, 127, 128, 254, 255, 256)
SLOT_CASES = [
    ('mini-sin-nocross-4-contiguous', 'lm_mini', 'sin', False, 4, False, 1500, CHECKPOINTS + (1502,)),
    ('mini-rope-nocross-4-paged', 'lm_mini', 'rope', False, 4, True, 1500, CHECKPOINTS + (1502,)),
    ('mini-sin_rope-nocross-40-contiguous', 'lm_mini', 'sin_rope', False, 40, False, 260, CHECKPOINTS),
    ('mini-sin-cross-4-paged', 'lm_mini', 'sin', True, 4, True, 260, CHECKPOINTS),
    ('mini-rope-cross-40-contiguous', 'lm_mini', 'rope', True, 40, False, 260, (0, 31, 64, 129)),
    ('mini-sin_rope-cross-4-contiguous', 'lm_mini', 'sin_rope', True, 4, False, 260, (0, 32, 63, 65, 256)),
    ('mini-sin-nocross-128-paged', 'lm_mini', 'sin', False, 128, True, 140, (0, 31, 64, 128)),
    ('tiny-sin-cross-4-contiguous', 'lm_tiny', 'sin', True, 4, False, 140, (0, 31, 64, 128)),
    ('medium-sin-cross-4-contiguous', 'lm_medium_2l', 'sin', True, 4, False, 70, (0, 32, 65)),
    ('large-rope-nocross-4-paged', 'lm_large_2l', 'rope', False, 4, True, 70, (0, 32, 65)),
    ('melody-sin-5-contiguous', 'lm_mini_melody', 'sin', False, 5, False, 260, CHECKPOINTS),
    ('melody-sin_rope-5-paged', 'lm_mini_melody', 'sin_rope', False, 5, True, 260, CHECKPOINTS),
]
# admission's cross K/V runs in chunks of 64 rows: 65 and 129 leave a 1-row last chunk, 150 a 22-row one
TEXT_LENS = (1, 31, 32, 33, 64, 65, 129, 150)
# condition prefixes of the melody cases, by slot: side by side in one session, on both sides of the first page boundary
PREFIXES = (9, 63, 64, 65, 0)


def _slot_offset(i, slots):
    """The step at which slot i is admitted: 0, 1, 31, 64 for the first four (their n then differ by 1, 31 and 64), the
    others spread over the first 70 steps; the last slot of a 4-slot session comes in at step 64, so the checkpoints before
    it see a slot never admitted."""
    return (0, 1, 31, 64)[i] if i < 4 else (7 * i) % 70


@pytest.mark.gpu
@pytest.mark.parametrize('case', SLOT_CASES, ids=[c[0] for c in SLOT_CASES])
def test_slot_step_matches_float64(case):
    """A SlotSession on the probe LM with staggered admissions (on lm_mini_melody each slot with its own condition prefix):
    at each checkpoint step every row's embedding, LayerNorm, q32, every layer's K / V at its own cache position (prefix +
    column), and the self- or cross-attention output, against float64; the cross K/V of every admission; and the cache
    positions the step changed."""
    from audiocraft_b200.batching import Request, SlotSession
    tag, name, pe, cross, slots, paged, gen_len, checkpoints = case
    melody = name == 'lm_mini_melody'
    cfg, sd0, m = _probe(name, pe, cross, prefix=melody)
    d, Hn, NL, K = cfg['dim'], cfg['num_heads'], cfg['num_layers'], cfg['n_q']
    w = m._w
    rows = 2 * slots
    max_prefix = max(PREFIXES) if melody else 0
    kv_pages = None
    if paged:   # room for every request plus free pages to poison
        from audiocraft_b200.batching import PagePool
        kv_pages = slots * PagePool.need(max_prefix + gen_len + 8) + 6
    sess = SlotSession(m, slots, gen_len, max_text=max(TEXT_LENS) if cross else 1, use_sampling=False, kv_pages=kv_pages,
                       max_prefix=max_prefix)
    b = m._bufs
    g = torch.Generator().manual_seed(slots + gen_len)
    T, Pfx = {}, {}
    admit_at = {}
    for i in range(slots):
        admit_at.setdefault(_slot_offset(i, slots), []).append(i)
    if cross:   # cache positions the admissions must not touch
        b['ck_cache'].fill_(NAN)
        b['cv_cache'].fill_(NAN)

    def admit(slot):
        Tt = TEXT_LENS[(slot * 3) % len(TEXT_LENS)] if cross else 0
        cr = (torch.randn(2, Tt, d, generator=g) * 0.5) if cross else None
        P = PREFIXES[slot % len(PREFIXES)] if melody else 0
        prefix = torch.randn(2, P, d, generator=g) * 0.5 if melody else None
        before = (b['ck_cache'].clone(), b['cv_cache'].clone()) if cross else None
        sess.admit(slot, Request(gen_len, cr, seed=slot, prefix=prefix))
        T[slot], Pfx[slot] = Tt, P
        if cross:
            torch.cuda.synchronize()
            for half in range(2):
                r = half * slots + slot
                c16 = cr[half].half().cuda()
                for layer in range(NL):
                    v64, bnd = gemm64(c16, w['w_ckv'][layer])
                    for j, nm in enumerate(('ck_cache', 'cv_cache')):
                        ref = v64[:, j * d:(j + 1) * d].reshape(Tt, Hn, 64).transpose(0, 1)
                        e = bnd[:, j * d:(j + 1) * d].reshape(Tt, Hn, 64).transpose(0, 1)
                        check_gemm_f16(b[nm][layer, r, :, :Tt], ref, e, f'{tag} admission slot {slot} T={Tt} layer {layer} {nm}')
            for j, nm in enumerate(('ck_cache', 'cv_cache')):
                keep = torch.ones_like(b[nm], dtype=torch.bool)
                keep[:, [slot, slots + slot], :, :Tt] = False
                assert bool(_nan_equal(b[nm], before[j])[keep].all()), f'{tag}: admission of slot {slot} wrote {nm} outside [0, T)'

    step = 0
    for cp in checkpoints:
        while step < cp:   # run up to the checkpoint, admitting on the way
            for s in admit_at.pop(step, []):
                admit(s)
            nxt = min([cp] + [t for t in admit_at if t > step])
            sess.steps(nxt - step)
            step = nxt
        for s in admit_at.pop(step, []):
            admit(s)
        _check_slot_step(sess, m, cfg, T, Pfx, f'{tag} step {step}', paged, cross)
        step += 1


def _check_slot_step(sess, m, cfg, T, Pfx, tag, paged, cross):
    """One step of the session, checked.  T / Pfx: each admitted slot's text and condition-prefix length; row r of slot
    r % slots reads its sequence at the slot's column and runs at cache position prefix + column, n = that position + 1."""
    b, w = m._bufs, m._w
    slots = sess.slots
    rows = 2 * slots
    d, Hn, NL = cfg['dim'], cfg['num_heads'], cfg['num_layers']
    st = sess.status()
    cols = torch.tensor([c for c, _ in st])[torch.arange(rows) % slots]              # per row, the slot's column
    pos = cols + torch.tensor([Pfx.get(s, 0) for s in range(slots)])[torch.arange(rows) % slots]   # cache position
    active_slot = torch.tensor([s == 1 for _, s in st])
    active = active_slot[torch.arange(rows) % slots]
    n = pos + 1
    seq = b['seq'][torch.arange(rows) % slots, :, :].cpu()
    toks = seq[torch.arange(rows), :, cols]                                          # [rows, K]
    ridx = torch.arange(rows)

    # poison what the step must not read, snapshot the caches
    if paged:
        kp, vp, table = sess.k_pool, sess.v_pool, sess.page_table.cpu()
        if sess.pages.free:
            idx = torch.tensor(sess.pages.free, device='cuda')
            kp[:, idx] = NAN
            vp[:, idx] = NAN
        for r in range(rows):
            s = r % slots
            held = sess.pages.held.get(s)
            if held is None:
                continue
            if not bool(active[r]):
                ids = held[(r // slots) * len(held) // 2:(r // slots + 1) * len(held) // 2]
                kp[:, ids] = NAN
                vp[:, ids] = NAN
                continue
            p = int(pos[r])
            npg = len(held) // 2
            kp[:, table[r, p // PAGE], :, p % PAGE:] = NAN
            vp[:, table[r, p // PAGE], :, p % PAGE:] = NAN
            if p // PAGE + 1 < npg:
                kp[:, table[r, p // PAGE + 1:npg].long()] = NAN
                vp[:, table[r, p // PAGE + 1:npg].long()] = NAN
        kc, vc = kp, vp
    else:
        kc, vc = b['k_cache'], b['v_cache']
        for r in range(kc.shape[1]):
            if r >= rows or not bool(active[r]):
                kc[:, r] = NAN
                vc[:, r] = NAN
            else:
                kc[:, r, :, int(pos[r]):] = NAN
                vc[:, r, :, int(pos[r]):] = NAN
    if cross:
        for r in range(b['ck_cache'].shape[1]):
            Tt = T.get(r % slots, 0) if r < rows else 0
            b['ck_cache'][:, r, :, Tt:] = NAN
            b['cv_cache'][:, r, :, Tt:] = NAN
        ck0, cv0 = b['ck_cache'].clone(), b['cv_cache'].clone()
    k0, v0 = kc.clone(), vc.clone()

    sess.steps(1)
    torch.cuda.synchronize()

    # the caches: exactly position n - 1 of each active row, in every layer
    for name, now, then in (('k', kc, k0), ('v', vc, v0)):
        changed = ~_nan_equal(now, then)
        want = torch.zeros_like(changed)
        for r in range(rows):
            if bool(active[r]):
                p = int(pos[r])
                if paged:
                    want[:, int(table[r, p // PAGE]), :, p % PAGE] = True
                else:
                    want[:, r, :, p] = True
        assert torch.equal(changed, want), f'{tag}: the step changed {name} cache positions other than n - 1 of active rows'
    if cross:
        assert bool(_nan_equal(b['ck_cache'], ck0).all() and _nan_equal(b['cv_cache'], cv0).all()), f'{tag}: cross cache changed'

    def kv_at(layer, nm):
        c = kc if nm == 'k' else vc
        if paged:
            pg = table[ridx, pos // PAGE].long().cuda()
            return c[layer][pg, :, (pos % PAGE).cuda()]
        return c[layer][ridx.cuda(), :, pos.cuda()]

    x0, tol = embed64(w, cfg, toks, pos)
    check(b['x'][:rows], x0, tol, f'{tag} lm_embed_slot_kernel')
    check_ln(b['h16'][:rows], b['x'][:rows], w['out_norm'][0], w['out_norm'][1], f'{tag} lm_ln_kernel d={d}')
    h = b['h16'][:rows]
    act = ridx[active]
    check_qkv(m, cfg, h[act.cuda()], pos[act], lambda l, nm: kv_at(l, nm)[act.cuda()],
              f'{tag} lm_qkv_slot{"_paged" if paged else ""}_kernel', b['q32'][:rows][act.cuda()])
    a16 = b['a16'][:rows]
    if cross:
        assert not bool(a16[[r for r in range(rows) if T.get(r % slots, 0) == 0]].any()), f'{tag}: slot never admitted'
        groups = []
        for Tt in sorted(set(T.values())):
            rr = torch.tensor([r for r in range(rows) if T.get(r % slots, 0) == Tt])
            if len(rr):
                groups.append((rr.cuda(), b['ck_cache'][-1][rr.cuda(), :, :Tt], b['cv_cache'][-1][rr.cuda(), :, :Tt]))
        check_attention(a16, h.view(rows, Hn, 64), groups, f'{tag} lm_cross_attn_slot_kernel', cross=True)
    else:
        assert not bool(a16[(~active).cuda()].any()), f'{tag}: rows of slots not decoding must be exactly 0'
        q = b['q32'][:rows].half().view(rows, Hn, 64)
        groups = []
        for nn in sorted(set(n[active].tolist())):
            rr = ridx[active & (n == nn)]
            if paged:
                pgs = table[rr][:, :-(-nn // PAGE)].long().cuda()                                  # [R, pages]
                kk = kc[-1][pgs].permute(0, 2, 1, 3, 4).reshape(len(rr), Hn, -1, 64)[:, :, :nn]
                vv = vc[-1][pgs].permute(0, 2, 1, 3, 4).reshape(len(rr), Hn, -1, 64)[:, :, :nn]
            else:
                kk, vv = kc[-1][rr.cuda(), :, :nn], vc[-1][rr.cuda(), :, :nn]
            groups.append((rr.cuda(), kk, vv))
        check_attention(a16, q, groups, f'{tag} lm_attn2_slot{"_paged" if paged else ""}_kernel')


# ----------------------------------------------------------------------------- contiguous decode step (generate)

KEY_COUNTS = (1, 2, 31, 32, 33, 63, 64, 65, 128, 129, 255, 256, 257, 1503)
# (id, model, pe, cross attention, batch, rows per item (1: no CFG, 2: CFG, 3: double CFG), key counts)
GEN_CASES = [
    ('mini-sin-B6', 'lm_mini', 'sin', False, 6, 1, KEY_COUNTS),
    ('mini-rope-B1', 'lm_mini', 'rope', False, 1, 1, KEY_COUNTS),
    ('mini-sin_rope-B32', 'lm_mini', 'sin_rope', False, 32, 1, (1, 33, 64, 257)),
    ('mini-sin-B100', 'lm_mini', 'sin', False, 100, 1, (1, 32, 65, 256, 1503)),
    ('tiny-sin-B32', 'lm_tiny', 'sin', False, 32, 1, (2, 63, 129)),
    ('mini-sin-cross-B1-text65', 'lm_mini', 'sin', True, 1, 2, (1, 65, 1503)),
    ('mini-rope-cross-B6-text33-cfg2', 'lm_mini', 'rope', True, 6, 3, (2, 129)),
    ('mini-sin_rope-cross-B100-text150', 'lm_mini', 'sin_rope', True, 100, 2, (31, 256)),
    ('medium-sin-cross-B6-text32', 'lm_medium_2l', 'sin', True, 6, 2, (33, 257)),
    ('large-rope-B6', 'lm_large_2l', 'rope', False, 6, 1, (64, 257)),
]
FOLD_CASES = ('mini-sin-B6', 'tiny-sin-B32')   # the FF2 (K = 4 d) has ACB_LM_MAX_SPLIT K slices at d = 128, 256


@pytest.mark.gpu
@pytest.mark.parametrize('case', GEN_CASES, ids=[c[0] for c in GEN_CASES])
def test_generate_step_matches_float64(case):
    """The generate() decode step (streaming_begin / streaming_step, acb_lm_step_logits) at key counts n: caches [0, n - 1)
    random, NaN from n - 1 on; every row's embedding, LayerNorm, q32 and K / V of every layer at position n - 1, and the self-
    or cross-attention output against float64; the cross K/V written by acb_lm_begin; the residual fold bit for bit."""
    tag, name, pe, cross, B, per, counts = case
    cfg, sd0, m = _probe(name, pe, cross)
    d, Hn, NL, K = cfg['dim'], cfg['num_heads'], cfg['num_layers'], cfg['n_q']
    w = m._w
    rows = B * per
    Tt = int(tag.split('text')[1].split('-')[0]) if cross else 0
    g = torch.Generator().manual_seed(B * 31 + Tt)
    max_len = max(counts) + 1
    cr = (torch.randn(rows, Tt, d, generator=g) * 0.5) if cross else None
    m._ensure(rows, max_len + 1, Tt, B)
    b = m._bufs
    if cross:
        b['ck_cache'].fill_(NAN)
        b['cv_cache'].fill_(NAN)
    m.streaming_begin(B, cr, max_len, cfg_coef_beta=1.5 if per == 3 else None)
    b = m._bufs
    torch.cuda.synchronize()
    if cross:   # EPI_CROSSKV at acb_lm_begin: rows [0, rows), positions [0, T); nothing past T
        c16 = cr.reshape(rows * Tt, d).half().cuda()
        for layer in range(NL):
            v64, bnd = gemm64(c16, w['w_ckv'][layer])
            for j, nm in enumerate(('ck_cache', 'cv_cache')):
                ref = v64[:, j * d:(j + 1) * d].reshape(rows, Tt, Hn, 64).transpose(1, 2)
                e = bnd[:, j * d:(j + 1) * d].reshape(rows, Tt, Hn, 64).transpose(1, 2)
                check_gemm_f16(b[nm][layer, :rows, :, :Tt], ref, e, f'{tag} acb_lm_begin layer {layer} {nm}')
                assert bool(torch.isnan(b[nm][:, :, :, Tt:]).all() and torch.isnan(b[nm][:, rows:]).all()), \
                    f'{tag}: acb_lm_begin wrote {nm} outside rows x [0, T)'
    ridx = torch.arange(rows)
    for nk in counts:
        p = nk - 1
        toks = torch.randint(-1, cfg['card'] + 2, (B, K), generator=g)
        for name_ in ('k_cache', 'v_cache'):
            c = b[name_]
            c.fill_(NAN)
            if p:
                c[:, :rows, :, :p] = (torch.randn(NL, rows, Hn, p, 64, generator=g) * 0.7).half().cuda()
        k0, v0 = b['k_cache'].clone(), b['v_cache'].clone()
        b['pos'][0] = p
        m.streaming_step(toks)
        torch.cuda.synchronize()
        t = f'{tag} n={nk}'
        for nm, then in (('k_cache', k0), ('v_cache', v0)):
            changed = ~_nan_equal(b[nm], then)
            want = torch.zeros_like(changed)
            want[:, :rows, :, p] = True
            assert torch.equal(changed, want), f'{t}: the step changed {nm} positions other than n - 1'
        x0, tol = embed64(w, cfg, toks.clamp(max=cfg['card'] + 1)[ridx % B], torch.full((rows,), p))
        check(b['x'][:rows], x0, tol, f'{t} lm_embed_kernel<false>')
        check_ln(b['h16'][:rows], b['x'][:rows], w['out_norm'][0], w['out_norm'][1], f'{t} lm_ln_kernel d={d}')
        h = b['h16'][:rows]
        check_qkv(m, cfg, h, torch.full((rows,), p), lambda l, nm: b[f'{nm}_cache'][l, :rows, :, p], f'{t} EPI_QKV',
                  b['q32'][:rows])
        if cross:
            check_attention(b['a16'][:rows], h.view(rows, Hn, 64),
                            [(ridx.cuda(), b['ck_cache'][-1][:rows, :, :Tt], b['cv_cache'][-1][:rows, :, :Tt])],
                            f'{t} lm_cross_attn_kernel<false>', cross=True)
        else:
            for r0 in range(0, rows, 32):
                rr = ridx[r0:r0 + 32].cuda()
                check_attention(b['a16'][:rows], b['q32'][:rows].half().view(rows, Hn, 64),
                                [(rr, b['k_cache'][-1][rr, :, :nk], b['v_cache'][-1][rr, :, :nk])],
                                f'{t} lm_attn2_kernel<false>')
        if tag in FOLD_CASES and nk == counts[1]:
            _check_fold_step(m, cfg, sd0, b, rows, p, toks, t)


def _check_fold_step(m, cfg, sd0, b, rows, p, toks, tag):
    """The same step again with the last layer's linear2 put back: x_B = ((x_A + p0) + p1) + ... over the `part` slots
    bit for bit, and those slots add up to that FF2."""
    last, d = cfg['num_layers'] - 1, cfg['dim']
    xa = b['x'][:rows].clone()
    wl = sd0[f'transformer.layers.{last}.linear2.weight'].half().cuda()
    m._w['w_ff2'][last].copy_(wl)
    try:
        b['pos'][0] = p
        m.streaming_step(toks)
        torch.cuda.synchronize()
    finally:
        m._w['w_ff2'][last].zero_()
    pad = _nt_rows_pad(rows)
    flat = b['part'].view(-1)
    parts = [flat[s * pad * d:s * pad * d + rows * d].view(rows, d) for s in range(_lib.ACB_LM_MAX_SPLIT)]
    v64, bnd = gemm64(b['f16'][:rows], wl)
    check(sum(pp.double() for pp in parts), v64, bnd, f'{tag} FF2 in the {_lib.ACB_LM_MAX_SPLIT} part slots')
    check_fold(b['x'][:rows], xa, parts, f'{tag} lm_ln_kernel residual fold')
    check_ln(b['h16'][:rows], b['x'][:rows], m._w['out_norm'][0], m._w['out_norm'][1], f'{tag} lm_ln_kernel after the fold')


# ----------------------------------------------------------------------------- prefill passes

def _check_pass(m, cfg, tag, R, p0, tc, x_ref, kv, ck=None, zeroed=(0, 0)):
    """The buffers after the last prefill pass, whose rows are (token, row) pairs r = tok * R + j at positions p0 + tok:
    x against x_ref(pos, j), the LayerNorm, q32 and every layer's K / V at each row's position (kv(layer, j) -> the
    generation row's K, V [H, positions, 64] read back), and the output of self attention over [0, pos] or, with ck(j) ->
    (K, V) [H, T, 64], of cross attention.  Rows in [zeroed[0], zeroed[1]) of h16 / a16 were zeroed after the passes (the
    decode step's padded rows): their LayerNorm, K / V and attention are not readable."""
    b, w = m._bufs, m._w
    Hn, NL = cfg['num_heads'], cfg['num_layers']
    M = R * tc
    pos, j = p0 + torch.arange(M) // R, torch.arange(M) % R
    x0, tol = x_ref(pos, j)
    check(b['x'][:M], x0, tol, f'{tag} embedding')
    keep = torch.tensor([r for r in range(M) if not zeroed[0] <= r < zeroed[1]])
    kc = keep.cuda()
    pos, j, n = pos[keep], j[keep], len(keep)
    h, a16, q32 = b['h16'][:M][kc], b['a16'][:M][kc], b['q32'][:M][kc]
    check_ln(h, b['x'][:M][kc], w['out_norm'][0], w['out_norm'][1], f'{tag} lm_ln_kernel')
    full = {(l, jj): kv(l, jj) for l in range(NL) for jj in range(R)}

    def kv_at(layer, nm):
        return torch.stack([full[(layer, int(j[r]))][nm == 'v'][:, int(pos[r])] for r in range(n)])
    check_qkv(m, cfg, h, pos, kv_at, f'{tag} pass QKV', q32)
    if ck is not None:
        groups = []
        for jj in range(R):
            rr = torch.nonzero(j == jj).flatten()
            k, v = ck(jj)
            groups.append((rr.cuda(), k.expand(len(rr), *k.shape), v.expand(len(rr), *v.shape)))
        check_attention(a16, h.view(n, Hn, 64), groups, f'{tag} lm_cross_attn_kernel<true>', cross=True)
    else:
        q = q32.half().view(n, Hn, 64)
        groups = [(torch.tensor([r]).cuda(), *(t[:, :int(pos[r]) + 1].unsqueeze(0) for t in full[(NL - 1, int(j[r]))]))
                  for r in range(n)]
        check_attention(a16, q, groups, f'{tag} causal pass attention')


def _last_pass(start, n, R):
    per = _lib.ACB_LM_PREFILL_ROWS // R
    done = (n - 1) // per * per
    return start + done, n - done


# (id, model, pe, cross, batch (contiguous) or None (an admission), prefix length P, prompt columns F)
PREFILL_CASES = [
    ('contiguous-rope-B1', 'lm_mini', 'rope', False, 1, 0, 100),
    ('contiguous-sin-B2-cross', 'lm_mini', 'sin', True, 2, 0, 33),
    ('contiguous-sin_rope-B3-cross', 'lm_tiny', 'sin_rope', True, 3, 0, 50),
    ('paged-rope-P0-F33', 'lm_mini', 'rope', False, None, 0, 33),
    ('paged-sin-cross-P0-F40', 'lm_mini', 'sin', True, None, 0, 40),
    ('paged-melody-sin_rope-P9-F60', 'lm_mini_melody', 'sin_rope', False, None, 9, 60),
    ('melody-sin-P63', 'lm_mini_melody', 'sin', False, None, 63, 0),
    ('melody-sin_rope-P64', 'lm_mini_melody', 'sin_rope', False, None, 64, 0),
    ('melody-sin-P65', 'lm_mini_melody', 'sin', False, None, 65, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize('case', PREFILL_CASES, ids=[c[0] for c in PREFILL_CASES])
def test_prefill_passes_match_float64(case):
    """The last prompt or prefix prefill pass, inspected right after the call: acb_lm_prefill after streaming_begin
    (contiguous-*), a paged admission with prompt columns (paged-*, the last pass spanning page 1 / 2 with P = 9, F = 60 and
    a single token with F = 33) and a melody admission's prefix passes (melody-*).  The caches are NaN before the call and
    afterwards hold exactly the positions the call fills."""
    from audiocraft_b200.batching import PagePool, Request, SlotSession
    tag, name, pe, cross, B, P, Fc = case
    cfg, sd0, m = _probe(name, pe, cross, prefix=P > 0)
    d, Hn, NL, K, card = cfg['dim'], cfg['num_heads'], cfg['num_layers'], cfg['n_q'], cfg['card']
    w = m._w
    g = torch.Generator().manual_seed(P * 100 + Fc)
    Tt = 33 if cross else 0

    if B is not None:   # acb_lm_prefill on a generation of B items (2 B rows with cross attention: CFG)
        rows = 2 * B if cross else B
        cr = (torch.randn(rows, Tt, d, generator=g) * 0.5) if cross else None
        m.streaming_begin(B, cr, Fc + 8)
        b = m._bufs
        b['k_cache'].fill_(NAN)
        b['v_cache'].fill_(NAN)
        seq = torch.randint(-1, card + 1, (B, K, Fc), generator=g)
        b['seq'][:B, :, :Fc] = seq.cuda()
        _lib.check(m._lib.acb_lm_prefill(m._handle, 0, Fc, _lib.stream()), 'lm_prefill')
        torch.cuda.synchronize()
        assert int((~torch.isnan(b['k_cache'])).sum()) == NL * rows * Hn * Fc * 64, f'{tag}: K written outside [0, F)'
        p0, tc = _last_pass(0, Fc, rows)

        def x_ref(pos, j):
            return embed64(w, cfg, seq[j % B, :, pos], pos)
        ck = (lambda jj: (b['ck_cache'][-1][jj, :, :Tt], b['cv_cache'][-1][jj, :, :Tt])) if cross else None
        _check_pass(m, cfg, tag, rows, p0, tc, x_ref, lambda l, jj: (b['k_cache'][l, jj], b['v_cache'][l, jj]), ck,
                    zeroed=(rows, _nt_rows_pad(rows)))
        return

    # an admission into slot 1 of a 4-slot session: its rows are cache / table rows 1 and 5
    slots, slot, gen_len = 4, 1, Fc + 20
    paged = tag.startswith('paged')
    kv_pages = slots * PagePool.need(P + gen_len + 8) if paged else None
    sess = SlotSession(m, slots, gen_len, max_text=64 if cross else 1, use_sampling=False, max_prefix=65 if P else 0,
                       kv_pages=kv_pages)
    b = m._bufs
    kc, vc = (sess.k_pool, sess.v_pool) if paged else (b['k_cache'], b['v_cache'])
    kc.fill_(NAN)
    vc.fill_(NAN)
    prefix = torch.randn(2, P, d, generator=g) * 0.5 if P else None
    cr = torch.randn(2, Tt, d, generator=g) * 0.5 if cross else None
    prompt = torch.randint(0, card, (1, K, Fc + 4), generator=g) if Fc else None
    sess.admit(slot, Request(gen_len, cr, prompt, seed=3, prefix=prefix, prefill_cols=Fc))
    torch.cuda.synchronize()
    n_pos = P + Fc
    assert int((~torch.isnan(kc)).sum()) == NL * 2 * Hn * n_pos * 64, f'{tag}: K written outside the slot\'s [0, P + F)'
    crow = (slot, slots + slot)
    if paged:
        table = sess.page_table.cpu()

        def kv(layer, jj):
            pg = table[crow[jj], :-(-n_pos // PAGE)].long().cuda()
            return tuple(c[layer][pg].permute(1, 0, 2, 3).reshape(Hn, -1, 64) for c in (kc, vc))
    else:
        def kv(layer, jj):
            return kc[layer, crow[jj]], vc[layer, crow[jj]]
    ck = (lambda jj: (b['ck_cache'][-1][crow[jj], :, :Tt], b['cv_cache'][-1][crow[jj], :, :Tt])) if cross else None
    if Fc:
        seq_row = b['seq'][slot].cpu()
        p0, tc = _last_pass(P, Fc, 2)

        def x_ref(pos, j):
            return embed64(w, cfg, seq_row[:, pos - P].t(), pos)
    else:
        p0, tc = _last_pass(0, P, 2)

        def x_ref(pos, j):
            x = prefix[j, pos].half().double().cuda()
            return _add_sin(x, torch.zeros_like(x), w, cfg, pos)
    _check_pass(m, cfg, tag, 2, p0, tc, x_ref, kv, ck)
