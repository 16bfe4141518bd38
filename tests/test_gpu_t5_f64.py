"""Each T5 encoder kernel (csrc/t5.cu) against float64, computed from the kernel's own fp32 / fp16 inputs.

test_gpu_t5.py compares the conditioner end to end with the reference after 12 or 24 layers, at 1e-2 on the hidden states.
That bound absorbs a factor of 2 from a missing TF32 rounding, a relative bias of the wrong sign, and any norm-weight
indexing error while every norm weight is 1 (as in the synthetic weights and the golden).  Here acb_t5_encode runs with a
workspace the test owns (0xFF bytes, NaN in fp16 and fp32; `out` / `hidden` NaN), and every stage is compared with a float64
restatement of its operation on the inputs it read, read back from that workspace.

Probe weights.  w_o and w_fo are zero in every layer, so the residual stream stays the embedding (adding +-0 is exact).
final_ln is random, of both signs, with magnitudes 0.1-4, and layer l's norm j is 2^e(l, j) * final_ln with a distinct
exponent per (layer, sublayer) (NORM_EXP).  A power of two commutes with the kernel's g * (x * rs) and with TF32 rounding, so
the input of the last layer's sublayer j is exactly 2^e(L-1, j) * h, h being the final norm's output left in the workspace:
a norm read at a wrong offset (the other sublayer's, another layer's, final_ln) scales a GEMM input by a power of two.  The
layers' weights differ, so a wrong stacked-weight row offset fails too.  GEMM weights and proj_w are TF32-rounded first, as
T5Encoder does.  Two more calls put back only the last layer's w_o, then only its w_fo: x - emb is then that one GEMM
(FE_RESID, K = d and K = d_ff).

TF32 rounding.  The device rounds with cvt.rna.tf32.f32: to nearest, ties away from zero (tf32_rna here).  The host's
t5.round_tf32, used for the weights, rounds ties to even; values the device writes are compared with the device's rule.

Bounds (u = 2^-24).
  GEMM: TF32 x TF32 products (11-bit significands) are exact in fp32, so every fp32 summation order meets
    |got - ref| <= (K - 1) u sum_k |a_k w_k|; FE_QKV adds half an fp16 ulp of its fp16 output, FE_RELU half a TF32 ulp of
    its output (the ulp at |ref| + bound, which covers a rounding flip within the GEMM bound), FE_PROJ and FE_RESID one
    fp32 rounding (the bias add; x = fp32(emb + acc)).  Masked projection rows must be exact zeros.
  RMSNorm: the sum of squares is a tree of at most 14 fp32 roundings deep (4 fmaf per thread, 5 warp levels, 5 block levels),
    then / d and + eps, rsqrtf (2 ulp) and two products: 14 u |ref| to first order; the bound is 16 u |ref|.  h must equal
    tf32_rna(hidden) bit for bit.
  Attention: a score is an fp32 sum of 64 fp16 products, then + bias and - the running max, each rounded:
    E = 63 u sum_d |q_d k_d| + 2 u (|s + b| + max |s + b|) per key.  Logits within E of the exact ones move every softmax
    weight by a factor within exp(+-2 E), so the output by at most expm1(2 max E) max|v|.  On top: 2^-10 max|v| for the
    fp16 P (2^-11) with room for __expf and the fp32 sums of P.V and of the row sum (T u, well under 2^-11 at T <= 300),
    plus half a TF32 ulp of the output.  max|v| is over the row's unmasked keys.  A row with no unmasked key must be
    exactly 0.  Every element of h, a and f must be TF32-exact.
  Every check prints its worst element's fraction of its bound.  Worst fractions over all cases on an H100 80GB HBM3 (700 W
  power limit): RMSNorm 0.26; FE_PROJ 0.04 and FE_RESID 0.04, except where the fp32 rounding of x dominates the bound (0.31
  with the embedding x 1e3, 0.74 at K = 4); attention 0.31.  FE_QKV 0.96 and FE_RELU 0.95 are their own output rounding
  (half an fp16 / TF32 ulp).  The TF32 wgmma's fp32 accumulation stays far inside the round-to-nearest bound, so the
  bound is not widened.

Coverage: the kernel instances and the case ids of test_t5_stages_match_float64 that run each against float64.
  t5_embed_kernel                                      every case (ids 0 and vocab - 1 included)
  t5_rmsnorm_kernel                                    every case, after each of the three calls; d 64 (16 of 512 threads
                                                       live) up to 2048 (all 512): min, wide; embedding x 1e3: hot
  lm_fwd_gemm_kernel<TF32, FE_QKV>                     every case; N tails (576 = 4 x 128 + 64): ragged, (192): min
  lm_fwd_attn_kernel<FA_T5>                            every case:
      T = 1: min; T on the 64 tiles: wide (64); off them: small (65), large (63), hot (129), ragged (130)
      T > max_distance (saturated buckets), 5 query tiles: base (300); num_buckets 16 != H 3, max_distance 20: ragged;
      H == num_buckets: wide; first key tile fully masked then unmasked keys (the corr path from -inf), a mask with
      holes, a fully masked item: ragged; length-1 items: small, large, min; grid z = 33: small; scores near +-100: hot
  lm_fwd_gemm_kernel<TF32, FE_RESID>  K = d            every case; N tail (192): ragged; N below one tile (64): min
                                      K = d_ff         every case; K tail inside a 32-float chunk (300 = 9 x 32 + 12):
                                                       ragged; K below one chunk (4): min
  lm_fwd_gemm_kernel<TF32, FE_RELU>                    every case; N tail (300): ragged; N below one box (4): min
  lm_fwd_gemm_kernel<TF32, FE_PROJ>                    every case; N tail (100): ragged; N below one box (4): min
  M = 2145 (items straddle 128-row tiles): small
"""
import ctypes as C
import math

import pytest
import torch

from audiocraft_b200 import t5 as T5
from tests.test_gpu_kernels_f64 import U, check, gemm64, half_ulp16

EPS = 1e-6
VOCAB = 1000
NORM_EXP = ((2, -3), (-1, 2), (1, -2))   # e(l, j): layer l's norm j is 2^e(l, j) * final_ln
ATTN_SLACK = 2.0 ** -10
NORM_BOUND_U = 16

# id -> shapes, B x T and the leading items' mask lengths (the rest random; None: the masks built in inputs())
CASES = {
    'small': dict(d=512, ff=2048, out=1536, L=2, B=33, T=65, lengths=[65, 1]),
    'base': dict(d=768, ff=3072, out=1536, L=3, B=2, T=300, lengths=[300, 217]),
    'large': dict(d=1024, ff=4096, out=1536, L=2, B=5, T=63, lengths=[63, 40, 17, 62, 1]),
    'ragged': dict(d=192, ff=300, out=100, L=2, B=4, T=130, nb=16, max_distance=20, lengths=None),
    'min': dict(d=64, ff=4, out=4, L=1, B=1, T=1, lengths=[1]),
    'wide': dict(d=2048, ff=512, out=2048, L=2, B=2, T=64, lengths=[64, 40]),
    'hot': dict(d=768, ff=3072, out=1536, L=2, B=2, T=129, lengths=[129, 100], emb_scale=1e3, q_scale=40.0),
}


# ----------------------------------------------------------------------------- TF32 rounding and float64 references

def tf32_rna(t: torch.Tensor) -> torch.Tensor:
    """fp32 values rounded to TF32 as cvt.rna.tf32.f32 does: to nearest, ties away from zero (finite values)."""
    b = t.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def tf32_trunc(t: torch.Tensor) -> torch.Tensor:
    return (t.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def half_ulp_tf32(a: torch.Tensor) -> torch.Tensor:
    """Half the spacing of TF32 numbers (10 stored mantissa bits) at magnitude |a|."""
    e = torch.floor(torch.log2(a.double().abs().clamp(min=2.0 ** -126)))
    return torch.exp2(e - 11)


def assert_tf32_exact(t: torch.Tensor, what: str):
    low = t.float().contiguous().view(torch.int32) & 0x1FFF
    n = int(low.count_nonzero())
    assert n == 0, f'{what}: {n} of {t.numel()} elements are not TF32 values (low 13 mantissa bits set)'


def assert_rna_of(h: torch.Tensor, hidden: torch.Tensor, what: str):
    """h is tf32_rna(hidden) bit for bit."""
    want = tf32_rna(hidden).view(torch.int32)
    bad = h.float().contiguous().view(torch.int32) != want
    if bool(bad.any()):
        i = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f'{what}: {int(bad.sum())} elements differ from the ties-away TF32 rounding of the fp32 '
                             f'output; first at {i}: {float(h[i])!r} vs {float(tf32_rna(hidden)[i])!r}')


def check_norm(hidden, h, x, g, what: str):
    """hidden = g * x * rsqrt(mean(x^2) + eps) within NORM_BOUND_U u; h = tf32_rna(hidden), TF32-exact."""
    x64 = x.double()
    ref = g.double() * x64 / torch.sqrt((x64 * x64).mean(-1, keepdim=True) + float(torch.tensor(EPS, dtype=torch.float32)))
    check(hidden, ref, NORM_BOUND_U * U * ref.abs(), f'{what}: RMSNorm')
    assert_rna_of(h, hidden, f'{what}: RMSNorm h')
    assert_tf32_exact(h, f'{what}: RMSNorm h')


def check_qkv(o, v64, bnd, d: int, what: str):
    B, Hn, T, _ = o['q'].shape
    for i, n in enumerate('qkv'):
        r = v64[..., i * d:(i + 1) * d].reshape(B, T, Hn, 64).transpose(1, 2)
        b = bnd[..., i * d:(i + 1) * d].reshape(B, T, Hn, 64).transpose(1, 2)
        check(o[n], r, b + half_ulp16(r.abs() + b), f'{what}: FE_QKV {n}')


def check_relu(got, v64, bnd, what: str):
    r = v64.clamp(min=0)
    check(got, r, bnd + half_ulp_tf32(r + bnd), f'{what}: FE_RELU')
    assert_tf32_exact(got, f'{what}: FE_RELU')


def check_proj(got, v64, bnd, bias, mask, what: str):
    live = mask.bool().unsqueeze(-1)
    ref = (v64 + bias.double()) * live
    tol = (bnd + U * ((v64 + bias.double()).abs() + bnd)) * live   # masked rows: 0, i.e. exact zeros
    check(got, ref, tol, f'{what}: FE_PROJ')


def check_resid(x, emb, v64, bnd, what: str):
    check(x.double() - emb.double(), v64, bnd + U * x.double().abs(), what)


def t5_bias(rel_bias: torch.Tensor, buckets: torch.Tensor, T: int) -> torch.Tensor:
    """[H, T, T]: bias[h, i, j] = rel_bias[buckets[j - i + T - 1], h]."""
    i = torch.arange(T, device=rel_bias.device)
    return rel_bias[buckets.long()[i.view(1, -1) - i.view(-1, 1) + T - 1]].permute(2, 0, 1)


def attn64_t5(q, k, v, rel_bias, buckets, mask):
    """float64 softmax(q k^T + bias) v over the unmasked keys of fp16 q / k / v [B, H, T, 64]; a row without one is 0.
    Returns (out [B, T, H * 64], tol) with the bound of the module docstring (0 on rows without a key)."""
    B, Hn, T, _ = q.shape
    q64, k64, v64 = q.double(), k.double(), v.double()
    s = q64 @ k64.transpose(-1, -2) + t5_bias(rel_bias.double(), buckets, T)
    keep = mask.bool().view(B, 1, 1, T).expand(B, Hn, T, T)
    live = keep.any(-1, keepdim=True)
    p = torch.where(live, torch.softmax(s.masked_fill(~keep, -math.inf), -1), torch.zeros_like(s))
    o = p @ v64
    sb = s.abs().masked_fill(~keep, 0.0)
    e = 63 * U * (q64.abs() @ k64.abs().transpose(-1, -2)) + 2 * U * (sb + sb.amax(-1, keepdim=True))
    e = e.masked_fill(~keep, 0.0).amax(-1, keepdim=True)
    vmax = v64.abs().amax(-1).view(B, Hn, 1, T).expand(B, Hn, T, T).masked_fill(~keep, 0.0).amax(-1, keepdim=True)
    tol = ((ATTN_SLACK + torch.expm1(2 * e)) * vmax).expand_as(o)
    tol = torch.where(live, tol + half_ulp_tf32(o.abs() + tol), torch.zeros_like(tol))

    def flat(t):
        return t.permute(0, 2, 1, 3).reshape(B, T, Hn * 64)
    return flat(o), flat(tol)


def check_attn(o, rel_bias, buckets, mask, what: str):
    ref, tol = attn64_t5(o['q'], o['k'], o['v'], rel_bias, buckets, mask)
    check(o['a'], ref, tol, f'{what}: FA_T5 attention')
    assert_tf32_exact(o['a'], f'{what}: FA_T5 attention')


# ----------------------------------------------------------------------------- probe weights and inputs

def case_shapes(name: str) -> dict:
    c = dict(CASES[name])
    c.setdefault('nb', 32)
    c.setdefault('max_distance', 128)
    c['H'] = c['d'] // 64
    return c


def probe_weights(c: dict, seed: int) -> dict:
    """Full weights (w_o / w_fo included) on the CPU: the probe zeroes w_o and w_fo, the FE_RESID calls restore one."""
    g = torch.Generator().manual_seed(seed)
    d, ff, H, L, out = c['d'], c['ff'], c['H'], c['L'], c['out']

    def n(*shape, std):
        return torch.randn(*shape, generator=g) * std
    final_ln = torch.where(torch.rand(d, generator=g) < 0.5, -1.0, 1.0) * \
        torch.exp(math.log(0.1) + torch.rand(d, generator=g) * math.log(40.0))
    w = dict(shared=n(VOCAB, d, std=c.get('emb_scale', 1.0)),
             w_qkv=T5.round_tf32(torch.cat([n(L, d, d, std=c.get('q_scale', 1.0) * (d * 64) ** -0.5),
                                            n(L, d, d, std=d ** -0.5), n(L, d, d, std=d ** -0.5)], 1)),
             w_o=T5.round_tf32(n(L, d, d, std=d ** -0.5)),
             w_i=T5.round_tf32(n(L, ff, d, std=d ** -0.5)),
             w_fo=T5.round_tf32(n(L, d, ff, std=ff ** -0.5)),
             ln=torch.stack([torch.stack([final_ln * 2.0 ** NORM_EXP[li][j] for j in (0, 1)]) for li in range(L)]),
             final_ln=final_ln,
             rel_bias=n(c['nb'], H, std=1.5),
             proj_w=T5.round_tf32(n(out, d, std=d ** -0.5)),
             proj_b=n(out, std=0.5))
    return w


def variant(w: dict, keep: str = None) -> dict:
    """The probe: w_o and w_fo zero in every layer except, when `keep` names one of them, its last layer."""
    v = dict(w)
    for name in ('w_o', 'w_fo'):
        z = torch.zeros_like(w[name])
        if name == keep:
            z[-1] = w[name][-1]
        v[name] = z
    return v


def inputs(name: str, c: dict, seed: int):
    """(ids [B, T], mask [B, T], buckets [2T - 1] int32) on the CPU."""
    g = torch.Generator().manual_seed(seed)
    B, T = c['B'], c['T']
    ids = torch.randint(0, VOCAB, (B, T), generator=g)
    ids[0, 0] = VOCAB - 1
    ids.view(-1)[-1] = 0
    if c['lengths'] is None:   # ragged: holes after a fully masked first key tile, one fully masked item
        mask = torch.ones(B, T, dtype=torch.long)
        mask[0, :64] = 0
        mask[0, 64::5] = 0
        mask[1] = 0
        mask[3, 70:] = 0
    else:
        lengths = list(c['lengths']) + torch.randint(1, T + 1, (B - len(c['lengths']),), generator=g).tolist()
        mask = (torch.arange(T).view(1, -1) < torch.tensor(lengths).view(-1, 1)).long()
    buckets = T5.relative_position_buckets(T, c['nb'], c['max_distance'])
    return ids, mask, buckets


def layout(c: dict) -> dict:
    """acb_t5_encode's workspace: x, h fp32 [M][d]; q, k, v fp16 [B][H][T][64]; a fp32 [M][d]; f fp32 [M][d_ff]; each
    256-byte aligned, M = B T."""
    M, d = c['B'] * c['T'], c['d']
    out, off = {}, 0
    for name, nbytes in [('x', M * d * 4), ('h', M * d * 4), ('q', M * d * 2), ('k', M * d * 2), ('v', M * d * 2),
                         ('a', M * d * 4), ('f', M * c['ff'] * 4)]:
        out[name] = off
        off += (nbytes + 255) // 256 * 256
    out['total'] = off
    return out


def abi_config(c: dict):
    from audiocraft_b200 import _lib
    return _lib.T5Config(c['d'], 64, c['H'], c['L'], c['ff'], VOCAB, c['nb'], c['out'], EPS)


# ----------------------------------------------------------------------------- the stage checks

def check_probe(o: dict, c: dict, w: dict, ids, mask, buckets, tag: str):
    """The probe call: embedding, final RMSNorm, the last layer's FE_QKV, FA_T5 and FE_RELU, and FE_PROJ."""
    e0, e1 = NORM_EXP[c['L'] - 1]
    assert torch.equal(o['x'], w['shared'][ids]), f'{tag}: x is not shared[ids] (embedding, or a non-zero residual add)'
    check_norm(o['hidden'], o['h'], o['x'], w['final_ln'], tag)
    v64, bnd = gemm64(o['h'] * 2.0 ** e0, w['w_qkv'][-1])
    check_qkv(o, v64, bnd, c['d'], tag)
    check_attn(o, w['rel_bias'], buckets, mask, tag)
    v64, bnd = gemm64(o['h'] * 2.0 ** e1, w['w_i'][-1])
    check_relu(o['f'], v64, bnd, tag)
    v64, bnd = gemm64(o['h'], w['proj_w'])
    check_proj(o['out'], v64, bnd, w['proj_b'], mask, tag)


def check_resid_call(o: dict, w: dict, keep: str, tag: str):
    """w_o (K = d) or w_fo (K = d_ff) of the last layer alone: x - emb is that GEMM of the call's own a or f."""
    src = 'a' if keep == 'w_o' else 'f'
    emb = w['shared'][o['ids']]
    v64, bnd = gemm64(o[src], w[keep][-1])
    check_resid(o['x'], emb, v64, bnd, f'{tag}: FE_RESID {keep} (K = {o[src].shape[-1]})')
    check_norm(o['hidden'], o['h'], o['x'], w['final_ln'], f'{tag} with {keep}')


# ----------------------------------------------------------------------------- CPU emulation of the kernels (self-test)

def emulate(c: dict, w: dict, ids, mask, buckets, attn_bias=None, attn_mask=None, ff2_input=None, h_round=tf32_rna):
    """acb_t5_encode's arithmetic on the CPU: fp32 / TF32 operands, fp32 GEMM sums, fp16 q / k / v and P, ties-away TF32
    rounding of every activation.  The keyword arguments inject one mistake: the attention's bias [H, T, T] or key mask,
    a change to FF2's input, the rounding of the norm output."""
    B, T, d, H = c['B'], c['T'], c['d'], c['H']
    eps = torch.tensor(EPS, dtype=torch.float32)
    x = w['shared'][ids].clone()
    bias = t5_bias(w['rel_bias'], buckets, T) if attn_bias is None else attn_bias
    amask = mask if attn_mask is None else attn_mask
    st = {}

    def norm(g):
        rs = torch.rsqrt((x * x).sum(-1, keepdim=True) / d + eps)
        y = g * (x * rs)
        return h_round(y), y

    def heads(t):
        return t.view(B, T, H, 64).transpose(1, 2).contiguous().half()
    for li in range(c['L']):
        h, _ = norm(w['ln'][li][0])
        qkv = h @ w['w_qkv'][li].t()
        q, k, v = heads(qkv[..., :d]), heads(qkv[..., d:2 * d]), heads(qkv[..., 2 * d:])
        s = q.float() @ k.float().transpose(-1, -2) + bias
        s = s.masked_fill(~amask.bool().view(B, 1, 1, T), -math.inf)
        m = s.amax(-1, keepdim=True)
        p = torch.exp(s - m).nan_to_num(nan=0.0)
        lsum = p.sum(-1, keepdim=True)
        o = (p.half().float() @ v.float()) * torch.where(lsum > 0, 1.0 / lsum, torch.zeros_like(lsum))
        a = tf32_rna(o.transpose(1, 2).reshape(B, T, d))
        x = x + a @ w['w_o'][li].t()
        h, _ = norm(w['ln'][li][1])
        f = tf32_rna((h @ w['w_i'][li].t()).clamp(min=0))
        fin = f if ff2_input is None else ff2_input(f)
        x = x + fin @ w['w_fo'][li].t()
        st.update(q=q, k=k, v=v, a=a, f=f)
    h, hidden = norm(w['final_ln'])
    out = (h @ w['proj_w'].t() + w['proj_b']) * mask.unsqueeze(-1)
    return dict(st, x=x, h=h, hidden=hidden, out=out, ids=ids)


def test_float64_checks_accept_kernel_arithmetic_and_reject_mutations():
    """CPU: every check accepts an fp32 / TF32 emulation of the kernel arithmetic on the 'ragged' and 'min' cases, and
    rejects a transposed relative bias, the bias of head h + 1, a masked key left unmasked, a zeroed 32-float K chunk of
    FF2, TF32 truncation of the norm output, ties-to-even on a tie, and a layer norm off by a power of two or read from the
    other sublayer.  The restated workspace layout equals acb_t5_workspace_bytes for every case."""
    # the ties-away rule itself
    one = torch.tensor([1 + 2.0 ** -11, -(1 + 2.0 ** -11), 1 + 3 * 2.0 ** -11, 1 + 2.0 ** -12, 3.0])
    assert tf32_rna(one).tolist() == [1 + 2.0 ** -10, -(1 + 2.0 ** -10), 1 + 2.0 ** -9, 1.0, 3.0]
    assert T5.round_tf32(one).tolist() == [1.0, -1.0, 1 + 2.0 ** -9, 1.0, 3.0]

    for name in ('ragged', 'min'):
        c = case_shapes(name)
        w = probe_weights(c, 3)
        ids, mask, buckets = inputs(name, c, 4)
        probe = variant(w)
        o = emulate(c, probe, ids, mask, buckets)
        check_probe(o, c, probe, ids, mask, buckets, f'self-check {name}')
        for keep in ('w_o', 'w_fo'):
            wk = variant(w, keep)
            check_resid_call(emulate(c, wk, ids, mask, buckets), wk, keep, f'self-check {name}')

    c = case_shapes('ragged')
    w = probe_weights(c, 3)
    ids, mask, buckets = inputs('ragged', c, 4)
    probe = variant(w)
    T = c['T']
    rev = buckets.flip(0)   # bucket of i - j at index j - i + T - 1
    unmasked = mask.clone()
    unmasked[0, 5] = 1
    attn_mutations = {'transposed relative bias': dict(attn_bias=t5_bias(probe['rel_bias'], rev, T)),
                      'bias of head h + 1': dict(attn_bias=t5_bias(probe['rel_bias'].roll(-1, 1), buckets, T)),
                      'one masked key attended': dict(attn_mask=unmasked)}
    for what, kw in attn_mutations.items():
        o = emulate(c, probe, ids, mask, buckets, **kw)
        with pytest.raises(AssertionError):
            check_attn(o, probe['rel_bias'], buckets, mask, what)

    wfo = variant(w, 'w_fo')

    def cut(f):
        f = f.clone()
        f[..., 256:288] = 0
        return f
    with pytest.raises(AssertionError):
        check_resid_call(emulate(c, wfo, ids, mask, buckets, ff2_input=cut), wfo, 'w_fo', 'FF2 chunk zeroed')

    o = emulate(c, probe, ids, mask, buckets, h_round=tf32_trunc)
    with pytest.raises(AssertionError):
        check_norm(o['hidden'], o['h'], o['x'], probe['final_ln'], 'TF32 truncation')
    tie = o['hidden'].clone()
    tie[0, 0, 0] = 1 + 2.0 ** -11
    with pytest.raises(AssertionError):
        assert_rna_of(T5.round_tf32(tie), tie, 'ties to even')

    for what, ln in (('norm exponent off by one', lambda t: t[-1, 0].mul_(2.0)),
                     ('sublayer norms swapped', lambda t: t.copy_(t.flip(1)))):
        bad = dict(probe, ln=probe['ln'].clone())
        ln(bad['ln'])
        o = emulate(c, bad, ids, mask, buckets)
        with pytest.raises(AssertionError):
            check_probe(o, c, probe, ids, mask, buckets, what)

    from audiocraft_b200 import _lib, build
    build.build()
    L = _lib.lib()
    for name in CASES:
        c = case_shapes(name)
        assert L.acb_t5_workspace_bytes(C.byref(abi_config(c)), c['B'], c['T']) == layout(c)['total'], name


# ----------------------------------------------------------------------------- on the device

def encode(c: dict, w: dict, ids, mask, buckets) -> dict:
    """acb_t5_encode with this test's workspace (0xFF bytes) and NaN-filled out / hidden; views of every buffer."""
    from audiocraft_b200 import _lib
    L = _lib.lib()
    B, T, d, H = c['B'], c['T'], c['d'], c['H']
    lay = layout(c)
    conf = abi_config(c)
    n = L.acb_t5_workspace_bytes(C.byref(conf), B, T)
    assert n == lay['total']
    ws = torch.full((n,), 0xFF, dtype=torch.uint8, device='cuda')
    out = torch.full((B, T, c['out']), math.nan, device='cuda')
    hidden = torch.full((B, T, d), math.nan, device='cuda')
    wts = _lib.T5Weights(*[_lib.ptr(w[k]) for k in ('shared', 'w_qkv', 'w_o', 'w_i', 'w_fo', 'ln', 'final_ln', 'rel_bias',
                                                     'proj_w', 'proj_b')])
    _lib.check(L.acb_t5_encode(C.byref(conf), C.byref(wts), _lib.ptr(ids), _lib.ptr(mask), _lib.ptr(buckets), B, T,
                               _lib.ptr(out), _lib.ptr(hidden), _lib.ptr(ws), n, _lib.stream()), 't5_encode')
    torch.cuda.synchronize()

    def view(name, dtype, shape):
        nbytes = math.prod(shape) * torch.finfo(dtype).bits // 8
        return ws[lay[name]:lay[name] + nbytes].view(dtype).view(shape)
    return dict(x=view('x', torch.float32, (B, T, d)), h=view('h', torch.float32, (B, T, d)),
                q=view('q', torch.float16, (B, H, T, 64)), k=view('k', torch.float16, (B, H, T, 64)),
                v=view('v', torch.float16, (B, H, T, 64)), a=view('a', torch.float32, (B, T, d)),
                f=view('f', torch.float32, (B, T, c['ff'])), out=out, hidden=hidden, ids=ids)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_t5_stages_match_float64(name):
    c = case_shapes(name)
    w = {k: t.cuda().contiguous() for k, t in probe_weights(c, 11).items()}
    ids, mask, buckets = (t.cuda() for t in inputs(name, c, 12))
    tag = f'{name} d={c["d"]} ff={c["ff"]} B={c["B"]} T={c["T"]}'
    probe = variant(w)
    o = encode(c, probe, ids, mask, buckets)
    check_probe(o, c, probe, ids, mask, buckets, tag)
    if name == 'hot':
        s = (o['q'].double() @ o['k'].double().transpose(-1, -2)).abs().max()
        print(f'{tag}: max |q k| {float(s):.1f}')
        assert s > 50, 'the hot case no longer reaches large attention logits'
    for keep in ('w_o', 'w_fo'):
        wk = variant(w, keep)
        check_resid_call(encode(c, wk, ids, mask, buckets), wk, keep, tag)
