"""Each LM forward stage and each decode GEMM instance against float64, computed from the kernel's own fp16 / fp32 inputs.

The end-to-end tests compare logits after several layers with the fp16-emulating oracle at rtol 2e-2 / atol 3e-2; that
tolerance absorbs fp16 rounding flips compounded over layers, and with them errors such as a rotary angle one position off,
a causal mask off by one key or one missing K chunk.  Here every output of one kernel is compared with a float64 restatement
of that kernel's operation on the inputs it actually read, read back from buffers the caller owns: the workspace of
acb_lm_forward and the buffers of acb_lm_debug_gemms (the decode step's GEMMs alone).

Probe weights (forward).  A synthetic LM whose self / cross out-projections and linear2 are zero in every layer and whose
norm1 / norm_cross / norm2 are copies of out_norm: the residual stream stays exactly the embedding (adding +-0 is exact), so
the out-norm output left in the workspace's h16 is, bit for bit, the input of every layer's QKV, cross-q and FF1 GEMM.  The
layers' weights differ (2 or 3 layers), so a wrong stacked-weight row offset gives a wrong result, and the last layer's N-tail
tiles run against real rows of the next layer or the end of the matrix.  Two more calls put the last layer's out-projection
(cross out-projection when the model has cross attention), then its linear2, back: x_final - x0 is then that one GEMM
(FE_RESID).  The workspace is filled with 0xFF bytes (NaN in fp16 and fp32) and the logits with NaN before each call.

Bounds.  fp16 x fp16 products are exact in fp32, so any fp32 summation order meets |got - ref| <= (K - 1) 2^-24 sum_k |a_k w_k|
(GEMM_BOUND_FACTOR times that); an fp16 output adds half an fp16 ulp.  Where the kernel rounds to fp16 before an fp32 function
(rotary positions, GELU) the reference is the function of the fp16-rounded float64 product, and the tolerance adds what the
rounding can flip to within the GEMM bound.  Attention: 2^-10 max|v| over the attended keys of each head and row, plus half
an fp16 ulp (the kernel's fp16 P and __expf).  Every check prints its worst element's fraction of the bound.  On an H100 80GB
HBM3 the fp32 outputs of both wgmma GEMMs and of the mma.sync GEMM stayed within 0.08 of the round-to-nearest bound, so
GEMM_BOUND_FACTOR is 1; the fp16 outputs come near 1 through their own half-ulp rounding.

Coverage: the kernel instances, and the test here that runs each against float64.
  csrc/lm_forward.cu (one call runs every stage; ids of test_forward_stages_match_float64):
    lm_fwd_embed_kernel, sequence rows and prefix rows         every case; prefix rows: melody-rope-P9, melody-rope-P150
    lm_fwd_ln_kernel (out-norm)                               every case, after each of the three calls
    lm_fwd_gemm_kernel<FE_QKV>        self q / k / v           tiny-sin-B3-S64, large-sin-B3-S1
                                      self k / v beside cross q  mini-sin-B3-S65-text65, tiny-sin-B1-S1-text1,
                                                               ragged-sin-B3-S300-text64, medium-sin-B1-S64-text65
                                      cross q (N = d)          every case with cross attention
    lm_fwd_gemm_kernel<FE_QKV_ROPE>                            mini-rope-B1-S300, ragged-rope-B1-S65, medium-rope-B3-S63,
                                      (k only, beside cross q) mini-sin_rope-B3-S63-text150, large-sin_rope-B1-S65-text1,
                                      positions after a prefix melody-rope-P9, melody-rope-P150
    lm_fwd_gemm_kernel<FE_CKV>                                 every case with cross attention (text 1, 64, 65, 150)
    lm_fwd_gemm_kernel<FE_RESID>      W_o (K = d)              every case without cross attention
                                      W_co (K = d)             every case with cross attention
                                      linear2 (K = ffn)        every case; ragged K (816 = 12 x 64 + 48): ragged-*
    lm_fwd_gemm_kernel<FE_GELU>                                every case; ragged N (816): ragged-*
    lm_fwd_gemm_kernel<FE_LOGITS>                              every case; ragged N (400): ragged-*
    lm_fwd_attn_kernel<true>  (causal) every case without cross attention: S 1, 63, 64, 65, 300, P + S up to 215
    lm_fwd_attn_kernel<false> (cross)  every case with cross attention: text 1, 64, 65, 150
    causal mask, bit for bit                                   test_forward_is_causal_bit_for_bit
  Decode GEMMs, through acb_lm_debug_gemms (ids of test_decode_gemms_match_float64; rows 2, 12, 24, 40, 64, 80, 200 in each).
  On a 132-SM H100 nt_for_rows gives NT = 1, 2, 4, 8, 8 at rows 2, 12, 24, 40, 64, and rows 80 / 200 run the wide GEMM at
  NPAD 128 / 256.  pick_split gives the non-reducing GEMMs one K slice (kslice = K) and pick_ft2 then needs N x K >= 2M,
  N / 32 >= 119 and a 32-feature slab 32 (2K + 64) + 16 + 512 (8 NT + 1) bytes <= 120 KB:
    lm_mini (d 256): no GEMM has 2M weights                    <1|2|4|8, QKV|QKV_ROPE|GELU|F32|PARTIAL, 1>
                                                               lm_mini-sin, lm_mini-rope
    lm_medium_2l (d 1536): QKV, FF1, heads (K = 1536): 103-117 KB at NT <= 4, 131 KB at NT 8
                                                               <1|2|4, QKV|GELU|F32, 2> lm_medium_2l-sin
                                                               <1|2|4, QKV_ROPE, 2> lm_medium_2l-rope
                                                               <8, QKV|QKV_ROPE|GELU|F32, 1> lm_medium_2l-sin / -rope
      out-proj / cross q / out (3 slices of 512): FT2 = 2 at every NT; FF2 (4 slices of 1536): FT2 = 2 at NT <= 4, 1 at 8
                                                               <*, PARTIAL, 2>, <8, PARTIAL, 1> lm_medium_2l-*
    lm_large_2l (d 2048): QKV, FF1, heads (K = 2048): 131 KB at NT 1   <*, QKV|QKV_ROPE|GELU|F32, 1> lm_large_2l-sin / -rope
      out-proj etc. (3 slices of 704): FT2 = 2; FF2 (6 slices of 1376): FT2 = 2 at NT <= 4, 1 at 8
    ACB_LM_FT32=0: every GEMM on 16-feature tiles                lm_medium_2l-sin-ft16
    <8, QKV_ROPE, 2> is selected at none of the released widths on 132 SMs (the NT = 8 slab does not fit at d = 1536).
  lm_gemm_wide_kernel<128|256, EPI>, K slices from pick_split_wide (clusters for QKV / FF1 / heads, part slots for PARTIAL):
    lm_mini: QKV, FF1, heads cluster 4; out-proj 4 slots, FF2 8           lm_mini-sin, lm_mini-rope
    lm_medium_2l: QKV, FF1 cluster 4, heads 1; out-proj 5 slots, FF2 5     lm_medium_2l-sin, lm_medium_2l-rope
    lm_large_2l: QKV cluster 4, FF1, heads 1; out-proj 4 slots, FF2 4     lm_large_2l-sin, lm_large_2l-rope
    No GEMM of these widths takes a cluster of 2.
  Per pass: every layer's K / V cache at the step's position (with rotary positions at that position), the last layer's q32
  (fp32), f16 (GELU), the FF2 partial sums (the probe zeroes W_o, W_cq and W_co, so the 16 `part` slots add up to FF2 alone)
  and the logits.  Live rows get random fp16 activations, pad rows NaN; the K / V caches are NaN except where the pass writes.
"""
import ctypes as C
import functools
import math

import pytest
import torch
import torch.nn.functional as F

from audiocraft_b200 import synth
from oracle import lm_oracle as LO
from tests.test_forward_host import _cfg
from tests.test_gpu_edges import _swap, assert_close

U = 2.0 ** -24
# Multiple of the round-to-nearest bound (K - 1) 2^-24 sum |a w| allowed to the tensor-core GEMMs.
GEMM_BOUND_FACTOR = 1.0
RAGGED = dict(dim=192, num_heads=3, hidden_scale=4.25, card=100)   # the forward tests' configuration with N and K tails


# ----------------------------------------------------------------------------- float64 references and bounds

def half_ulp16(a: torch.Tensor) -> torch.Tensor:
    """Half the spacing of fp16 numbers at magnitude |a| (2^-25 in the subnormal range)."""
    e = torch.floor(torch.log2(a.double().abs().clamp(min=2.0 ** -14)))
    return torch.exp2(e - 11)


def gemm64(a: torch.Tensor, w: torch.Tensor):
    """float64 a @ w^T of fp16 operands, and the bound every fp32 summation order of the exact products meets."""
    a64, w64 = a.double(), w.double()
    return a64 @ w64.t(), GEMM_BOUND_FACTOR * (a.shape[-1] - 1) * U * (a64.abs() @ w64.abs().t())


def check(got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor, what: str):
    """|got - ref| <= tol element-wise (a NaN fails); prints the worst element's fraction of its bound."""
    got = got.double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = (got - ref).abs()
    frac = torch.where(err == 0, torch.zeros_like(err), err / tol).nan_to_num(nan=math.inf)
    worst = float(frac.max())
    print(f'{what}: max err {float(err.nan_to_num(nan=math.inf).max()):.2e}, {worst:.3f} of the bound')
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f'{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound (worst {worst:.3g}); '
                             f'first at {i}: got {float(got[i])!r}, want {float(ref[i])!r} +- {float(tol[i]):.3g}')


def check_gemm_f16(got, v64, bnd, what):
    check(got, v64, bnd + half_ulp16(v64.abs() + bnd), what)


def _flip(v64, bnd):
    """fp16(v64) and how far fp16 of an fp32 value within bnd of v64 can be from it."""
    r = v64.float().half().double()
    lo, hi = (v64 - bnd).float().half().double(), (v64 + bnd).float().half().double()
    return r, torch.maximum((lo - r).abs(), (hi - r).abs())


def check_rope(got, v64, bnd, pos0, cfg: dict, f16_out: bool, what: str):
    """q / k [R, H, T, 64] with rotary positions pos0 .. pos0 + T - 1 (pos0 an int, or a tensor [R]: each row from its own
    position): the kernel rotates fp16(its fp32 sum) in fp32.  The reference is the oracle's fp32 rotation of fp16(v64); the
    tolerance adds the input flips (|cos|, |sin| <= 1 with positional_scale in [0, 1]), both sides' fp32 rotation error and,
    for an fp16 output, half an ulp."""
    r, dev = _flip(v64, bnd)
    rot = (lambda t, p: LO.rope_rotate(t, p, cfg['max_period'], cfg['positional_scale']))
    r32 = r.float().cpu()
    if isinstance(pos0, int):
        ref = rot(r32, pos0)
    else:
        ref = torch.cat([rot(r32[i:i + 1], int(p)) for i, p in enumerate(pos0.tolist())])
    ref = ref.to(v64.device).double()
    pair = dev.unflatten(-1, (32, 2)).sum(-1, keepdim=True).expand(*dev.shape[:-1], 32, 2).flatten(-2)
    mag = r.abs().unflatten(-1, (32, 2)).sum(-1, keepdim=True).expand(*dev.shape[:-1], 32, 2).flatten(-2)
    tol = pair + 8 * U * mag
    if f16_out:
        tol = tol + half_ulp16(ref.abs() + tol)
    check(got, ref, tol, what)


def gelu64(x):
    return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))


def check_gelu(got, v64, bnd, what):
    """f16 = fp16(gelu_erf(fp16(v))) with gelu_erf in fp32: the reference is gelu64(fp16(v64)); the tolerance adds GELU's
    change over the fp16 inputs within the GEMM bound, the fp32 GELU's error and half an fp16 ulp."""
    r, _ = _flip(v64, bnd)
    g = gelu64(r)
    lo, hi = gelu64((v64 - bnd).float().half().double()), gelu64((v64 + bnd).float().half().double())
    tol = torch.maximum((lo - g).abs(), (hi - g).abs()) + 8 * U * (r.abs() * (1 + r.abs()) + g.abs())
    check(got, g, tol + half_ulp16(g.abs() + tol), what)


def check_ln(got, x, gamma, beta, what):
    """fp16 LayerNorm (eps 1e-5, fp32 statistics) vs fp16(float64 LayerNorm of the same fp32 rows): at most one fp16 ulp."""
    ref = F.layer_norm(x.double(), (x.shape[-1],), gamma.double(), beta.double(), 1e-5).float().half().double()
    check(got, ref, 2 * half_ulp16(torch.maximum(ref.abs(), got.double().abs().nan_to_num(nan=0.0))), what)


def attn64(q, k, v, mask=None):
    """float64 softmax(q k^T / 8) v of fp16 q [B, H, Tq, 64], k / v [B, H, Tk, 64]; mask [Tq, Tk] True where a key is
    attended (None: every key).  Returns (out [B, Tq, H * 64], tol)."""
    B, Hn, Tq, _ = q.shape
    s = q.double() @ k.double().transpose(-1, -2) / 8.0
    vmax = v.double().abs().amax(-1).unsqueeze(-2).expand(B, Hn, Tq, k.shape[2])   # [B, H, Tq, Tk]
    if mask is not None:
        s = s.masked_fill(~mask, -math.inf)
        vmax = vmax.masked_fill(~mask, 0.0)
    o = (torch.softmax(s, -1) @ v.double()).permute(0, 2, 1, 3)                      # [B, Tq, H, 64]
    t = (2.0 ** -10 * vmax.amax(-1)).permute(0, 2, 1).unsqueeze(-1).expand_as(o)
    return o.reshape(B, Tq, Hn * 64), (t + half_ulp16(o.abs() + t)).reshape(B, Tq, Hn * 64)


def causal_mask(T: int, device='cpu'):
    return torch.ones(T, T, dtype=torch.bool, device=device).tril()


# ----------------------------------------------------------------------------- forward workspace

def fwd_layout(cfg: dict, B: int, P: int, S: int, text_len: int) -> dict:
    """acb_lm_forward's workspace: x fp32 [M][d], h16 / q / k / v / a16 fp16 [M][d], f16 [M][ffn], c16 / ck / cv fp16
    [B * text][d] (nothing without cross attention), each 256-byte aligned, M = B (P + S)."""
    d, ffn = cfg['dim'], int(cfg['hidden_scale'] * cfg['dim'])
    M, Mt = B * (P + S), B * text_len if cfg['cross_attention'] else 0
    out, off = {}, 0
    for name, nbytes in [('x', M * d * 4)] + [(n, M * d * 2) for n in ('h16', 'q', 'k', 'v', 'a16')] + \
            [('f16', M * ffn * 2)] + [(n, Mt * d * 2) for n in ('c16', 'ck', 'cv')]:
        out[name] = off
        off += (nbytes + 255) // 256 * 256
    out['total'] = off
    return out


def _forward(m, cfg, seq, cross, prefix, B, P, S, Tt):
    """acb_lm_forward with this test's workspace (0xFF bytes) and logits (NaN); returns views of the workspace's buffers."""
    from audiocraft_b200 import _lib
    L = m._lib
    lay = fwd_layout(cfg, B, P, S, Tt)
    acfg = m._config()
    n = L.acb_lm_forward_workspace_bytes(C.byref(acfg), B, P, S, Tt)
    assert n == lay['total']
    ws = torch.full((n,), 0xFF, dtype=torch.uint8, device='cuda')
    logits = torch.full((B, cfg['n_q'], S, cfg['card']), math.nan, device='cuda')
    _lib.check(L.acb_lm_forward(C.byref(acfg), C.byref(m._weights()), _lib.ptr(seq), _lib.ptr(cross), _lib.ptr(prefix), B, P,
                                S, Tt, _lib.ptr(logits), _lib.ptr(ws), n, _lib.stream()), 'lm_forward')
    torch.cuda.synchronize()
    d, Hn, T, ffn = cfg['dim'], cfg['num_heads'], P + S, int(cfg['hidden_scale'] * cfg['dim'])

    def view(name, dtype, shape):
        nbytes = math.prod(shape) * torch.finfo(dtype).bits // 8
        return ws[lay[name]:lay[name] + nbytes].view(dtype).view(shape)
    out = dict(x=view('x', torch.float32, (B, T, d)), h16=view('h16', torch.float16, (B, T, d)),
               q=view('q', torch.float16, (B, Hn, T, 64)), k=view('k', torch.float16, (B, Hn, T, 64)),
               v=view('v', torch.float16, (B, Hn, T, 64)), a16=view('a16', torch.float16, (B, T, d)),
               f16=view('f16', torch.float16, (B, T, ffn)), logits=logits)
    if Tt:
        out.update(c16=view('c16', torch.float16, (B, Tt, d)), ck=view('ck', torch.float16, (B, Hn, Tt, 64)),
                   cv=view('cv', torch.float16, (B, Hn, Tt, 64)))
    return out


@functools.lru_cache(maxsize=2)
def _synth(name: str, over: tuple, cross: bool, seed: int):
    cfg = synth.lm_config(name)
    cfg.update(dict(over))
    cfg['cross_attention'] = cross
    return cfg, synth.synth_lm_state_dict(cfg, seed=seed)


def probe_state_dict(cfg: dict, sd: dict, zero: tuple, norms_from_out_norm: bool) -> dict:
    """A copy of sd with the named per-layer matrices zero in every layer and, optionally, every layer norm = out_norm."""
    sd = dict(sd)
    for li in range(cfg['num_layers']):
        p = f'transformer.layers.{li}.'
        for n in zero:
            if p + n in sd:
                sd[p + n] = torch.zeros_like(sd[p + n])
        if norms_from_out_norm:
            for n in ('norm1', 'norm_cross', 'norm2'):
                if p + n + '.weight' in sd:
                    sd[p + n + '.weight'] = sd['out_norm.weight'].clone()
                    sd[p + n + '.bias'] = sd['out_norm.bias'].clone()
    return sd


# ----------------------------------------------------------------------------- CPU self-check

def test_float64_checks_accept_kernel_arithmetic_and_reject_mutations():
    """CPU: each check accepts its own fp32 / fp16 emulation of the kernel arithmetic and rejects swapped items or heads, a
    rotary position one off, the diagonal key dropped from the causal mask and one K chunk of 64 zeroed; the workspace
    layout restated above gives the library's total for the shapes of the GPU tests."""
    g = torch.Generator().manual_seed(0)
    cfg = dict(max_period=10000.0, positional_scale=1.0)
    a = torch.randn(6, 320, generator=g).half()
    w = (torch.randn(72, 320, generator=g) / 16).half()
    v64, bnd = gemm64(a, w)
    f32 = a.float() @ w.float().t()
    check(f32, v64, bnd, 'self-check fp32 GEMM')
    check_gemm_f16(f32.half(), v64, bnd, 'self-check fp16 GEMM')
    a_cut = a.clone()
    a_cut[:, 128:192] = 0
    f32_cut = a_cut.float() @ w.float().t()
    for fn, bad in ((check, _swap(f32, 2)), (check, f32_cut), (check_gemm_f16, f32_cut.half()),
                    (check_gelu, gelu64(f32_cut.half().double()).half())):
        with pytest.raises(AssertionError):
            fn(bad, v64, bnd, 'mutated')
    check_gelu(F.gelu(f32.half().float()).half(), v64, bnd, 'self-check GELU')

    # rotary positions: [R, H, T, 64] at positions 37 ..
    qa = torch.randn(2 * 3 * 64, 320, generator=g).half()
    v64, bnd = gemm64(qa, w[:64])
    v64, bnd = v64.view(2, 3, 64, 64), bnd.view(2, 3, 64, 64)
    kern = LO.rope_rotate((qa.float() @ w[:64].float().t()).view(2, 3, 64, 64).half().float(), 37, 1e4, 1.0)
    check_rope(kern.half(), v64, bnd, 37, cfg, True, 'self-check rope fp16')
    check_rope(kern, v64, bnd, 37, cfg, False, 'self-check rope fp32')
    shifted = LO.rope_rotate(v64.float().half().float(), 38, 1e4, 1.0)
    for bad in (shifted, _swap(kern, 0, dim=1)):
        with pytest.raises(AssertionError):
            check_rope(bad, v64, bnd, 37, cfg, False, 'mutated rope')

    # LayerNorm
    x = torch.randn(5, 192, generator=g) * 3 + 1
    gm, bt = 1 + 0.1 * torch.randn(192, generator=g), 0.05 * torch.randn(192, generator=g)
    check_ln(F.layer_norm(x, (192,), gm, bt, 1e-5).half(), x, gm, bt, 'self-check LayerNorm')
    with pytest.raises(AssertionError):
        check_ln(_swap(F.layer_norm(x, (192,), gm, bt, 1e-5).half(), 1), x, gm, bt, 'swapped rows')

    # attention: causal (keys 0 .. i) and cross (every key)
    B, Hn, T, Tk = 2, 3, 70, 9
    q = torch.randn(B, Hn, T, 64, generator=g).half()
    k = torch.randn(B, Hn, T, 64, generator=g).half()
    v = torch.randn(B, Hn, T, 64, generator=g).half()
    for mask, kk, vv, what in ((causal_mask(T), k, v, 'causal'), (None, k[:, :, :Tk], v[:, :, :Tk], 'cross')):
        ref, tol = attn64(q, kk, vv, mask)
        s = (q.float() @ kk.float().transpose(-1, -2)) / 8
        if mask is not None:
            s = s.masked_fill(~mask, -math.inf)
        kern = (torch.softmax(s, -1) @ vv.float()).permute(0, 2, 1, 3).reshape(B, T, Hn * 64)
        check(kern.half(), ref, tol, f'self-check {what} attention')
        with pytest.raises(AssertionError):
            check(_swap(kern.view(B, T, Hn, 64), 1, dim=2).reshape(B, T, Hn * 64).half(), ref, tol, 'swapped heads')
    ref, tol = attn64(q, k, v, causal_mask(T))
    dropped, _ = attn64(q, k, v, causal_mask(T) & ~torch.eye(T, dtype=torch.bool))   # the diagonal key left out
    with pytest.raises(AssertionError):
        check(dropped[:, 1:].half(), ref[:, 1:], tol[:, 1:], 'diagonal key dropped')

    # the workspace layout
    from audiocraft_b200 import _lib, build
    build.build()
    L = _lib.lib()
    for name, over, pe, Bn, S, Tt, P in FORWARD_CASES:
        c = synth.lm_config(name)
        c.update(over)
        c['cross_attention'] = Tt is not None
        acfg = _cfg(dim=c['dim'], num_heads=c['num_heads'], num_layers=c['num_layers'], ffn_dim=int(c['hidden_scale'] * c['dim']),
                    card=c['card'], cross_attention=int(Tt is not None),
                    positional_embedding=['sin', 'rope', 'sin_rope'].index(pe))
        assert L.acb_lm_forward_workspace_bytes(C.byref(acfg), Bn, P, S, Tt or 0) == fwd_layout(c, Bn, P, S, Tt or 0)['total']


# ----------------------------------------------------------------------------- forward, stage by stage

# (name, overrides, positional embedding, B, S, text_len (None: no cross attention), prefix length)
FORWARD_CASES = [
    ('lm_mini', (), 'sin', 3, 65, 65, 0),
    ('lm_mini', (), 'rope', 1, 300, None, 0),
    ('lm_mini', (), 'sin_rope', 3, 63, 150, 0),
    ('lm_tiny', (), 'sin', 1, 1, 1, 0),
    ('lm_tiny', (), 'sin', 3, 64, None, 0),
    ('lm_mini', tuple(RAGGED.items()), 'sin', 3, 300, 64, 0),
    ('lm_mini', tuple(RAGGED.items()), 'rope', 1, 65, None, 0),
    ('lm_medium_2l', (), 'sin', 1, 64, 65, 0),
    ('lm_medium_2l', (), 'rope', 3, 63, None, 0),
    ('lm_large_2l', (), 'sin_rope', 1, 65, 1, 0),
    ('lm_large_2l', (), 'sin', 3, 1, None, 0),
    ('lm_mini_melody', (), 'rope', 3, 63, None, 9),
    ('lm_mini_melody', (), 'rope', 1, 65, None, 150),
]


def _case_id(c):
    name, over, pe, B, S, Tt, P = c
    short = 'ragged' if over else {'lm_mini_melody': 'melody'}.get(name, name.replace('lm_', '').replace('_2l', ''))
    return f'{short}-{pe}-' + (f'P{P}' if P else f'B{B}-S{S}' + (f'-text{Tt}' if Tt else ''))


@pytest.mark.gpu
@pytest.mark.parametrize('case', FORWARD_CASES, ids=[_case_id(c) for c in FORWARD_CASES])
def test_forward_stages_match_float64(case):
    from audiocraft_b200.lm import LMModel
    name, over, pe, B, S, Tt, P = case
    cross_attn = Tt is not None
    cfg0, sd0 = _synth(name, over, cross_attn, 7)
    cfg = dict(cfg0, positional_embedding=pe)
    d, Hn, NL, K, card = cfg['dim'], cfg['num_heads'], cfg['num_layers'], cfg['n_q'], cfg['card']
    T, last, rope, sin = P + S, NL - 1, pe != 'sin', pe != 'rope'
    sd = probe_state_dict(cfg, sd0, ('self_attn.out_proj.weight', 'cross_attention.out_proj.weight', 'linear2.weight'), True)
    m = LMModel(sd, cfg, None, None)
    w = m._w
    g = torch.Generator().manual_seed(B * 1000 + S + P)
    seq = torch.randint(0, card + 1, (B, K, S), generator=g).cuda()
    cross = (torch.randn(B, Tt, d, generator=g) * 0.5).cuda() if cross_attn else None
    prefix = (torch.randn(B, P, d, generator=g) * 0.5).cuda() if P else None
    tag = _case_id(case)
    o = _forward(m, cfg, seq, cross, prefix, B, P, S, Tt or 0)

    # embedding: the residual stream is still x0
    x0 = torch.zeros(B, T, d, device='cuda')
    for kq in range(K):
        x0[:, P:] = x0[:, P:] + w['emb'][kq][seq[:, kq]].float()
    if P:
        x0[:, :P] = prefix.half().float()
    if sin:
        x0 = x0 + cfg['positional_scale'] * LO.sin_embedding(torch.arange(T).view(1, -1, 1), d, cfg['max_period']).cuda()
    assert_close(o['x'], x0, 0, 1e-5, f'{tag} embedding (final x)')
    if P and not sin:
        assert torch.equal(o['x'][:, :P], prefix.half().float()), 'prefix rows are not fp16(prefix)'
    x0 = o['x'].clone()

    def ln_and_logits(o, what):
        check_ln(o['h16'], o['x'], w['out_norm'][0], w['out_norm'][1], f'{tag} {what}: out-norm LayerNorm')
        v64, bnd = gemm64(o['h16'][:, P:], w['heads'])
        perm = (lambda t: t.view(B, S, K, card).permute(0, 2, 1, 3))
        assert not bool(torch.isnan(o['logits']).any()), 'logits left unwritten'
        check(o['logits'], perm(v64), perm(bnd), f'{tag} {what}: FE_LOGITS')

    ln_and_logits(o, 'probe')
    h = o['h16']

    def heads(t, n):   # [B, n, H * 64] -> [B, H, n, 64]
        return t.view(B, n, Hn, 64).permute(0, 2, 1, 3)

    # self q / k / v of the last layer
    v64, bnd = gemm64(h, w['w_qkv'][last])
    names = ('k', 'v') if cross_attn else ('q', 'k', 'v')
    for i, n in enumerate(('q', 'k', 'v')):
        if n not in names:
            continue
        r, b = heads(v64[..., i * d:(i + 1) * d], T), heads(bnd[..., i * d:(i + 1) * d], T)
        if rope and n != 'v':
            check_rope(o[n], r, b, 0, cfg, True, f'{tag} FE_QKV_ROPE {n}')
        else:
            check_gemm_f16(o[n], r, b, f'{tag} FE_QKV {n}')
    if cross_attn:
        assert torch.equal(o['c16'], cross.half()), 'c16 is not fp16(cross)'
        v64, bnd = gemm64(o['c16'], w['w_ckv'][last])
        check_gemm_f16(o['ck'], heads(v64[..., :d], Tt), heads(bnd[..., :d], Tt), f'{tag} FE_CKV k')
        check_gemm_f16(o['cv'], heads(v64[..., d:], Tt), heads(bnd[..., d:], Tt), f'{tag} FE_CKV v')
        v64, bnd = gemm64(h, w['w_cq'][last])
        check_gemm_f16(o['q'], heads(v64, T), heads(bnd, T), f'{tag} FE_QKV cross q')
        ref, tol = attn64(o['q'], o['ck'], o['cv'])
        check(o['a16'], ref, tol, f'{tag} cross attention')
    else:
        ref, tol = attn64(o['q'], o['k'], o['v'], causal_mask(T, 'cuda'))
        check(o['a16'], ref, tol, f'{tag} causal attention')
    v64, bnd = gemm64(h, w['w_ff1'][last])
    check_gelu(o['f16'], v64, bnd, f'{tag} FE_GELU')

    # FE_RESID: the last layer's (cross) out-projection, then its linear2, alone
    p = f'transformer.layers.{last}.'
    for key, src, wname in (('w_co' if cross_attn else 'w_o', 'a16',
                             p + ('cross_attention.out_proj.weight' if cross_attn else 'self_attn.out_proj.weight')),
                            ('w_ff2', 'f16', p + 'linear2.weight')):
        wl = sd0[wname].half().cuda()
        w[key][last].copy_(wl)
        o = _forward(m, cfg, seq, cross, prefix, B, P, S, Tt or 0)
        w[key][last].zero_()
        v64, bnd = gemm64(o[src], wl)
        # x_final = fp32(x0 + the kernel's sum): one more rounding of |x_final|
        check(o['x'].double() - x0.double(), v64, bnd + U * o['x'].double().abs(),
              f'{tag} FE_RESID {key} (K = {wl.shape[1]})')
        ln_and_logits(o, f'with {key}')


@pytest.mark.gpu
@pytest.mark.parametrize('name,pe,P', [('lm_mini', 'sin', 0), ('lm_mini_melody', 'rope', 9)])
def test_forward_is_causal_bit_for_bit(name, pe, P):
    """forward(seq)[..., :t] == forward(seq[..., :t]) == forward(seq with every token at or after t replaced)[..., :t]: rows are
    summed in a fixed order and masked keys get P = 0 exactly, so a key one past the causal boundary changes bits."""
    from audiocraft_b200.lm import LMModel
    cfg = synth.lm_config(name)
    cfg['positional_embedding'] = pe
    sd = synth.synth_lm_state_dict(cfg, seed=17)
    m = LMModel(sd, cfg, None, None)
    B, S = 2, 300
    g = torch.Generator().manual_seed(18)
    seq = torch.randint(0, cfg['card'] + 1, (B, cfg['n_q'], S), generator=g)
    other = torch.randint(0, cfg['card'] + 1, (B, cfg['n_q'], S), generator=g)
    kw = {}
    if cfg['cross_attention']:
        kw['cross_attention_src'] = torch.randn(B, 7, cfg['dim'], generator=g) * 0.5
    if P:
        kw['prefix'] = torch.randn(B, P, cfg['dim'], generator=g) * 0.5
    full = m.forward(seq, **kw)
    for t in (1, 55, 63, 64, 65, 128, 129, 299):
        short = m.forward(seq[..., :t], **kw)
        alt = seq.clone()
        alt[..., t:] = other[..., t:]
        changed = m.forward(alt, **kw)
        assert torch.equal(short, full[..., :t, :]), f't = {t}: forward of the first t positions differs'
        assert torch.equal(changed[..., :t, :], full[..., :t, :]), f't = {t}: tokens at or after t change earlier logits'
        assert not torch.equal(changed[..., t:, :], full[..., t:, :])
    print(f'{name} {pe} P={P}: causal bit for bit at t = 1 .. 299')


# ----------------------------------------------------------------------------- decode GEMMs

DECODE_ROWS = (2, 12, 24, 40, 64, 80, 200)


def _nt_rows_pad(rows: int) -> int:
    """The decode step's padded row count: 8 NT below 65 rows, the wide GEMM's NPAD above (split stride of `part`)."""
    if rows > 64:
        return 128 if rows <= 128 else 256
    return 8 * (1 if rows <= 8 else 2 if rows <= 16 else 4 if rows <= 32 else 8)


def _decode_pass(m, cfg, rows: int, pos: int, seed: int, tag: str):
    from audiocraft_b200 import _lib
    d, Hn, NL, ffn = cfg['dim'], cfg['num_heads'], cfg['num_layers'], int(cfg['hidden_scale'] * cfg['dim'])
    rope, last = cfg['positional_embedding'] != 'sin', NL - 1
    g = torch.Generator().manual_seed(seed)
    m.streaming_begin(rows // 2, torch.randn(rows, 3, d, generator=g) * 0.5, max_len=300)
    b, w = m._bufs, m._w
    h = torch.randn(rows, d, generator=g).half().cuda()
    for name, val in (('h16', h), ('a16', (torch.randn(rows, d, generator=g) * 0.3).half().cuda())):
        b[name].fill_(math.nan)
        b[name][:rows] = val
    for name in ('f16', 'q32', 'logits', 'k_cache', 'v_cache'):
        b[name].fill_(math.nan)
    b['part'].zero_()
    b['pos'][0] = pos
    nl = C.c_int(0)
    _lib.check(m._lib.acb_lm_debug_gemms(m._handle, _lib.stream(), C.byref(nl)), 'lm_debug_gemms')
    torch.cuda.synchronize()
    assert nl.value == NL * (4 + 2 * int(cfg['cross_attention'])) + 1
    tag = f'{tag} rows={rows}'

    for layer in range(NL):
        v64, bnd = gemm64(h, w['w_qkv'][layer])
        for i, n in ((0, 'q'), (1, 'k'), (2, 'v')):
            if n == 'q' and layer != last:
                continue
            got = b['q32'][:rows].view(rows, Hn, 1, 64) if n == 'q' else b[f'{n}_cache'][layer, :rows, :, pos:pos + 1]
            r = v64[:, i * d:(i + 1) * d].reshape(rows, Hn, 1, 64)
            e = bnd[:, i * d:(i + 1) * d].reshape(rows, Hn, 1, 64)
            what = f'{tag} layer {layer} {"q32" if n == "q" else n + " cache"}'
            if rope and n != 'v':
                check_rope(got, r, e, pos, cfg, n != 'q', what + ' (rope)')
            elif n == 'q':
                check(got, r, e, what)
            else:
                check_gemm_f16(got, r, e, what)
    for n in ('k_cache', 'v_cache'):   # nothing else of the caches is written
        assert int((~torch.isnan(b[n])).sum()) == NL * rows * Hn * 64, f'{tag}: {n} written outside position {pos}'
    v64, bnd = gemm64(h, w['w_ff1'][last])
    check_gelu(b['f16'][:rows], v64, bnd, f'{tag} f16 (GELU)')
    stride = _nt_rows_pad(rows) * d
    slots = b['part'].view(-1)[:16 * stride].view(16, -1, d)[:, :rows].double().sum(0)
    v64, bnd = gemm64(b['f16'][:rows], w['w_ff2'][last])
    check(slots, v64, bnd, f'{tag} FF2 partial sums (16 part slots)')
    v64, bnd = gemm64(h, w['heads'])
    check(b['logits'][:rows], v64, bnd, f'{tag} logits (F32)')


@pytest.mark.gpu
@pytest.mark.parametrize('name,pe,ft32', [
    ('lm_mini', 'sin', None), ('lm_mini', 'rope', None), ('lm_medium_2l', 'sin', None), ('lm_medium_2l', 'rope', None),
    ('lm_large_2l', 'sin', None), ('lm_large_2l', 'rope', None), ('lm_medium_2l', 'sin', '0')],
    ids=['lm_mini-sin', 'lm_mini-rope', 'lm_medium_2l-sin', 'lm_medium_2l-rope', 'lm_large_2l-sin', 'lm_large_2l-rope',
         'lm_medium_2l-sin-ft16'])
def test_decode_gemms_match_float64(monkeypatch, name, pe, ft32):
    """One acb_lm_debug_gemms pass per row count on LMModel's own buffers: every layer's K / V cache at the step's position,
    the last layer's q32 and f16, the FF2 partial sums and the logits against float64 of the activations written in."""
    from audiocraft_b200.lm import LMModel
    if ft32 is None:
        monkeypatch.delenv('ACB_LM_FT32', raising=False)
    else:
        monkeypatch.setenv('ACB_LM_FT32', ft32)
    cfg0, sd0 = _synth(name, (), True, 7)
    cfg = dict(cfg0, positional_embedding=pe)
    sd = probe_state_dict(cfg, sd0, ('self_attn.out_proj.weight', 'cross_attention.out_proj.weight'), False)
    for li in range(cfg['num_layers']):   # W_cq: the first d rows of the cross in-projection
        p = f'transformer.layers.{li}.cross_attention.in_proj_weight'
        sd[p] = sd[p].clone()
        sd[p][:cfg['dim']] = 0
    m = LMModel(sd, cfg, None, None)
    rows_list = DECODE_ROWS if ft32 is None else (2, 12, 24, 40)
    for i, rows in enumerate(rows_list):
        _decode_pass(m, cfg, rows, 300 - rows, 100 + i, f'{name} {pe}' + (' ft16' if ft32 else ''))
