"""The FP8 self-attention KV pool of a paged session on the host: page bytes and pages per budget, the refusals before any
device work, the e4m3 quantizer oracle against a float64 nearest-even search over all 256 codes, and an fp32 emulation of
lm_attn2_slot_paged_fp8_kernel's partition against the float64 attention bound on code x scale.

Quantizer (include/audiocraft_b200.h, acb_lm_begin_slots_paged_fp8): amax = max |x_j|, inv = 448 / amax, code_j =
e4m3(x_j * inv) rounded to nearest even and saturated at +-448, scale = amax / 448, every operation one fp32 rounding;
amax == 0 stores zero codes and a zero scale.  `quant_e4m3` is that in fp32 torch ops, which the GPU tests compare bit for
bit with the pool.

Attention (emulate_fp8_attn32).  Iteration k of warp w covers positions (k * 8 + w) * 8 + pg, pg = lane / 4; each of the 4
lanes of a position dots its 16 codes with q / 8 in an fp32 chain, the 4 partial sums add in a 2-level tree, and the sum is
multiplied by the K scale; the softmax weight times the V scale scales the V codes.  Against the float64 attention on
code x scale (tests/test_gpu_decode_f64.attn_decode64) the score has at most 19 roundings (< the 64 the bound allows), each
weight passes through one more rounding (the V scale product) and one more merge (8 position groups per warp, not 4) than
the fp16 kernel's, and each accumulator chain holds ceil(n / 64) keys: fp8_attn64 passes n_it + 2 and ceil(n / 64) + 1."""
import contextlib
import math
import types

import pytest
import torch

from audiocraft_b200 import _lib
from audiocraft_b200.batching import ContinuousGenerator, PagePool, SlotSession, kv_page_bytes, kv_pages_for_budget, \
    pattern_sequence
from tests.test_continuous_paged_host import _RefusingLM
from tests.test_gpu_decode_f64 import attn_decode64
from tests.test_gpu_kernels_f64 import check

PAGE = _lib.ACB_LM_KV_PAGE
E4M3_MAX = 448.0


# ----------------------------------------------------------------------------- the quantizer oracle

def quant_e4m3(x):
    """x [..., 64] fp32 -> (codes [..., 64] torch.float8_e4m3fn, scales [...] fp32), as the kernels quantize."""
    x = x.float()
    amax = x.abs().amax(-1)
    live = amax > 0
    inv = torch.where(live, torch.tensor(E4M3_MAX) / torch.where(live, amax, torch.ones_like(amax)), torch.zeros_like(amax))
    codes = (x * inv.unsqueeze(-1)).to(torch.float8_e4m3fn)
    codes = torch.where(live.unsqueeze(-1), codes.view(torch.uint8), torch.zeros_like(codes.view(torch.uint8)))
    return codes.view(torch.float8_e4m3fn), torch.where(live, amax / E4M3_MAX, torch.zeros_like(amax))


def dequant(codes, scales):
    return codes.float() * scales.float().unsqueeze(-1)


def _e4m3_table():
    """(bit patterns, float64 values) of the 254 finite e4m3 codes (0x7F and 0xFF are NaN)."""
    bits = torch.tensor([b for b in range(256) if b & 0x7F != 0x7F], dtype=torch.uint8)
    return bits, bits.view(torch.float8_e4m3fn).double()


def nearest_even64(y):
    """float64 round-to-nearest-even onto the finite e4m3 codes of y (fp32 products x * inv, any shape): the code at the
    least distance, on a tie the one whose bit pattern is even; beyond 448 the nearest finite code is +-448 (saturation).
    +0 and -0 tie for a zero product."""
    bits, vals = _e4m3_table()
    y64 = y.double().reshape(-1, 1)
    dist = (y64 - vals.unsqueeze(0)).abs()
    best = dist.min(1, keepdim=True).values
    cand = dist == best
    odd = (bits & 1).bool().unsqueeze(0).expand_as(cand)
    pick = torch.where(cand & ~odd, 1, 0) * 2 + cand.int()          # an even candidate first, then any candidate
    idx = pick.argmax(1)
    return bits[idx].view(torch.float8_e4m3fn).double().reshape(y.shape)   # the sign of a zero is not compared


def _check_quant(x, what):
    codes, scales = quant_e4m3(x)
    amax = x.float().abs().amax(-1)
    inv = torch.where(amax > 0, torch.tensor(E4M3_MAX) / amax.clamp_min(1e-45), torch.zeros_like(amax))
    want = nearest_even64(x.float() * inv.unsqueeze(-1))
    want = torch.where((amax > 0).unsqueeze(-1), want, torch.zeros_like(want))
    got = codes.double()
    bad = (got != want) | (torch.signbit(got) != torch.signbit(want)) & (want != 0)
    assert not bool(bad.any()), f'{what}: {int(bad.sum())} codes differ from the float64 nearest-even search'
    sc_want = torch.where(amax > 0, amax / E4M3_MAX, torch.zeros_like(amax))
    assert torch.equal(scales, sc_want), what
    return codes, scales


def test_quantizer_matches_nearest_even_search():
    g = torch.Generator().manual_seed(11)
    for sc in (1e-3, 1.0, 37.0, 1e4):
        _check_quant(torch.randn(300, 64, generator=g) * sc, f'random x{sc}')
    _check_quant(torch.rand(200, 64, generator=g) * torch.logspace(-6, 3, 64), 'random over 9 decades')

    # one-hot vectors: the hot element is the amax and codes to exactly +-448, the others to 0
    for v in (1e-30, 0.5, -3.0, 7e5):
        x = torch.zeros(64, 64)
        x[torch.arange(64), torch.arange(64)] = v
        codes, scales = _check_quant(x, f'one-hot {v}')
        assert torch.equal(codes.float().diagonal(), torch.full((64,), math.copysign(448.0, v)))
        assert float(codes.float().abs().sum()) == 64 * 448.0 and bool((scales == torch.tensor(abs(v)) / 448.0).all())

    # rounding ties: with amax = 448 (inv = 1 exactly) every midpoint between two adjacent finite codes below 448
    _, vals = _e4m3_table()
    pos = torch.unique(vals[vals >= 0]).float()
    mids = ((pos[:-1].double() + pos[1:].double()) / 2).float()
    assert torch.equal(mids.double(), (pos[:-1].double() + pos[1:].double()) / 2), 'the midpoints are exact in fp32'
    n = mids.numel()
    body = torch.zeros(-(-n // 63) * 63)
    body[:n] = mids
    x = torch.cat([torch.full((body.numel() // 63, 1), 448.0), body.view(-1, 63)], 1)
    codes, _ = _check_quant(torch.cat([x, -x]), 'ties')
    # nearest-even by hand for the first ties: 2^-10 -> 0, 3 2^-10 -> 2^-8, 1.0625 -> 1, 1.1875 -> 1.25
    y = torch.tensor([[448.0, 2.0 ** -10, 3 * 2.0 ** -10, 1.0625, 1.1875] + [0.0] * 59])
    assert quant_e4m3(y)[0].float()[0, :5].tolist() == [448.0, 0.0, 2.0 ** -8, 1.0, 1.25]

    # subnormal codes: k 2^-9 for k = 1 .. 7, and values between them
    sub = torch.arange(1, 64, dtype=torch.float32) * 2.0 ** -12
    x = torch.cat([torch.tensor([448.0]), sub]).unsqueeze(0)
    codes, _ = _check_quant(torch.cat([x, -x]), 'subnormals')
    assert bool((codes.view(torch.uint8)[0, 1:] & 0x78 == 0).sum() > 20), 'the vector exercises the subnormal codes'

    # the amax element maps to exactly +-448 on random vectors of either sign
    x = torch.randn(500, 64, generator=g) * 3
    codes, _ = quant_e4m3(x)
    j = x.abs().argmax(-1)
    hot = codes.float()[torch.arange(500), j]
    assert torch.equal(hot, torch.where(x[torch.arange(500), j] > 0, 448.0, -448.0))

    # the zero vector (and -0): zero codes, zero scale
    x = torch.zeros(2, 64)
    x[1] = -0.0
    codes, scales = _check_quant(x, 'zero vector')
    assert not bool(codes.view(torch.uint8).any()) and not bool(scales.any())


# ----------------------------------------------------------------------------- attention emulation and bound

def fp8_attn64(q, k, v):
    """attn_decode64 on dequantized K / V [R, H, n, 64] with the FP8 kernel's counts (module docstring)."""
    n = k.shape[2]
    it = -(-n // 64)
    return attn_decode64(q, k, v, it + 1, it + 2)


def emulate_fp8_attn32(q, kc, ks, vc, vs):
    """fp32 emulation of attn2_paged_fp8_body for one query: q [H, 64] (fp16 values), kc / vc [H, n, 64] code values,
    ks / vs [H, n] scales.  Keys pp = (k * 8 + warp) * 8 + pg, 4 lanes of 16 dims per key, an online softmax per (warp,
    group), the groups merged (xor 4, 8, 16: pg with pg ^ 1, ^ 2, ^ 4), then the warps in order."""
    Hn, n, _ = kc.shape
    n_it = -(-n // 64)
    pad = n_it * 64 - n
    z = torch.zeros(Hn, pad, 64)
    kp = torch.cat([kc.float(), z], 1).view(Hn, n_it, 8, 8, 4, 16)
    vp = torch.cat([vc.float(), z], 1).view(Hn, n_it, 8, 8, 64)
    ksp = torch.cat([ks.float(), torch.zeros(Hn, pad)], 1).view(Hn, n_it, 8, 8)
    vsp = torch.cat([vs.float(), torch.zeros(Hn, pad)], 1).view(Hn, n_it, 8, 8)
    live = (torch.arange(n_it * 64) < n).view(n_it, 8, 8)
    qs = (q.float() * 0.125).view(Hn, 1, 1, 4, 16)
    m = torch.full((Hn, 8, 8), -math.inf)
    l = torch.zeros(Hn, 8, 8)
    acc = torch.zeros(Hn, 8, 8, 64)
    for it in range(n_it):
        part = (qs * kp[:, it]).sum(-1)                                              # [H, 8, 8, 4]
        s = ((part[..., 0] + part[..., 1]) + (part[..., 2] + part[..., 3])) * ksp[:, it]
        mn = torch.maximum(m, s)
        corr, pw = torch.exp(m - mn), torch.exp(s - mn)
        upd = live[it].expand(Hn, 8, 8)
        l = torch.where(upd, l * corr + pw, l)
        pv = pw * vsp[:, it]
        acc = torch.where(upd.unsqueeze(-1), acc * corr.unsqueeze(-1) + pv.unsqueeze(-1) * vp[:, it], acc)
        m = torch.where(upd, mn, m)

    def merge(ma, la, aa, mb, lb, ab):
        mn = torch.maximum(ma, mb)
        ca = torch.where(ma == -math.inf, torch.zeros_like(ma), torch.exp(ma - mn))
        cb = torch.where(mb == -math.inf, torch.zeros_like(mb), torch.exp(mb - mn))
        return mn, la * ca + lb * cb, aa * ca.unsqueeze(-1) + ab * cb.unsqueeze(-1)
    for stride in (1, 2, 4):   # pg with pg ^ stride; the result stands at the lower group
        a = torch.arange(0, 8, 2 * stride)
        b = a + stride
        mm, ll, aa = merge(m[..., a], l[..., a], acc[..., a, :], m[..., b], l[..., b], acc[..., b, :])
        m, l, acc = m.clone(), l.clone(), acc.clone()
        m[..., a], l[..., a], acc[..., a, :] = mm, ll, aa
    mw, lw, aw = m[..., 0], l[..., 0], acc[..., 0, :]                                 # [H, 8 warps]
    mx = mw.amax(-1, keepdim=True)
    cw = torch.where(mw == -math.inf, torch.zeros_like(mw), torch.exp(mw - mx))
    lt, ot = torch.zeros(Hn), torch.zeros(Hn, 64)
    for wi in range(8):
        lt = lt + lw[:, wi] * cw[:, wi]
        ot = ot + aw[:, wi] * cw[:, wi].unsqueeze(-1)
    return (ot / lt.unsqueeze(-1)).half().reshape(Hn * 64)


def test_fp8_attention_bound_accepts_the_kernel_partition_and_rejects_mutations():
    """The emulation passes the float64 bound on code x scale at n = 1, 64, 65 and 1503, and fails it with the scale of the
    neighbouring position or head, the K scale on V, the scale dropped, one key missing or extra, and a page swapped."""
    g = torch.Generator().manual_seed(5)
    Hn, N = 4, 1536   # 24 pages
    q = torch.randn(Hn, 64, generator=g).half()
    # K / V with per-position magnitudes that differ, as real activations do
    mag = torch.exp(torch.randn(Hn, N, 1, generator=g) * 0.5)
    kc, ks = quant_e4m3(torch.randn(Hn, N, 64, generator=g) * mag)
    vc, vs = quant_e4m3(torch.randn(Hn, N, 64, generator=g) * mag.flip(1))
    for n in (1, 64, 65, 1503):
        ref, tol = fp8_attn64(q.unsqueeze(0), dequant(kc[:, :n], ks[:, :n]).unsqueeze(0),
                              dequant(vc[:, :n], vs[:, :n]).unsqueeze(0))
        got = emulate_fp8_attn32(q, kc[:, :n], ks[:, :n], vc[:, :n], vs[:, :n]).unsqueeze(0)
        check(got, ref, tol, f'fp8 attention emulation n={n}')
    n = 1503
    ref, tol = fp8_attn64(q.unsqueeze(0), dequant(kc[:, :n], ks[:, :n]).unsqueeze(0), dequant(vc[:, :n], vs[:, :n]).unsqueeze(0))
    last = (n - 1) // PAGE
    first = torch.arange(PAGE)
    perm_sw = torch.cat([last * PAGE + first, torch.arange(PAGE, last * PAGE), first[:n - last * PAGE]])
    K, V = (kc[:, :n], ks[:, :n]), (vc[:, :n], vs[:, :n])
    mutants = {
        "the neighbouring position's scale": ((kc[:, :n], ks[:, 1:n + 1]), (vc[:, :n], vs[:, 1:n + 1])),
        "the neighbouring head's scale": ((kc[:, :n], ks[:, :n].roll(1, 0)), (vc[:, :n], vs[:, :n].roll(1, 0))),
        'the K scale applied to V': (K, (vc[:, :n], ks[:, :n])),
        'the scale dropped': ((kc[:, :n], torch.ones_like(ks[:, :n])), V),
        'newest key missing': ((kc[:, :n - 1], ks[:, :n - 1]), (vc[:, :n - 1], vs[:, :n - 1])),
        'one extra key': ((kc[:, :n + 1], ks[:, :n + 1]), (vc[:, :n + 1], vs[:, :n + 1])),
        'page 0 swapped with the last page': ((kc[:, perm_sw], ks[:, perm_sw]), (vc[:, perm_sw], vs[:, perm_sw])),
    }
    for what, ((k_c, k_s), (v_c, v_s)) in mutants.items():
        with pytest.raises(AssertionError):
            check(emulate_fp8_attn32(q, k_c, k_s, v_c, v_s).unsqueeze(0), ref, tol, what)


# ----------------------------------------------------------------------------- page arithmetic and refusals

def test_fp8_page_bytes_and_pages_per_budget():
    small = types.SimpleNamespace(num_layers=24, dim=1024, num_heads=16)
    medium = types.SimpleNamespace(num_layers=48, dim=1536, num_heads=24)
    large = types.SimpleNamespace(num_layers=48, dim=2048, num_heads=32)
    for lm in (small, medium, large):
        assert kv_page_bytes(lm, 'fp8') == 64 * lm.num_layers * (2 * lm.dim + 8 * lm.num_heads)
        assert kv_page_bytes(lm) == kv_page_bytes(lm, 'fp16') == 64 * 4 * lm.num_layers * lm.dim
    assert kv_page_bytes(small, 'fp8') == 3342336 and kv_page_bytes(large, 'fp8') == 13369344
    assert kv_page_bytes(medium, 'fp8') == 10027008 and kv_page_bytes(medium) == 18874368
    # the bytes of 3008 fp16 pages hold 5662 fp8 pages (1.88x)
    budget = 3008 * kv_page_bytes(medium) / 1e9
    assert kv_pages_for_budget(medium, budget) == 3008
    assert kv_pages_for_budget(medium, budget, 'fp8') == 5662
    assert kv_pages_for_budget(large, 61.5, 'fp8') == math.floor(61.5e9 / 13369344)
    for bad in ('fp32', 'bf16', 'e4m3', None, 8):
        with pytest.raises(ValueError):
            kv_page_bytes(medium, bad)
        with pytest.raises(ValueError):
            kv_pages_for_budget(medium, 1.0, bad)


def _fake_model():
    lm = _RefusingLM()
    lm.num_heads = 1
    gp = dict(use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=3.0, two_step_cfg=False, cfg_coef_beta=None)
    return types.SimpleNamespace(lm=lm, generation_params=gp, max_duration=2.0, duration=1.0, frame_rate=50,
                                 _has_melody=False)


def test_fp8_refusals_before_device_work(monkeypatch):
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    m = _fake_model()
    for bad in ('fp32', 'bf16', 'int8', None, 'FP8'):
        with pytest.raises(ValueError, match='dtype'):
            ContinuousGenerator(m, slots=4, kv_cache_gb=1.0, kv_cache_dtype=bad)
        with pytest.raises(ValueError, match='dtype'):
            SlotSession(m.lm, 4, 100, kv_pages=1000, kv_dtype=bad)
    with pytest.raises(ValueError, match='kv_cache_gb'):
        ContinuousGenerator(m, slots=4, kv_cache_dtype='fp8')
    with pytest.raises(ValueError, match='kv_pages'):
        SlotSession(m.lm, 4, 100, kv_dtype='fp8')
    # a budget of the fp8 page size reaches the device where fp16 pages would not fit
    need = PagePool.need(pattern_sequence(m.lm, None, 100)[0].shape[-1])
    gb = (need + 0.5) * kv_page_bytes(m.lm, 'fp8') / 1e9
    with pytest.raises(ValueError, match='cannot hold one request'):
        ContinuousGenerator(m, slots=4, kv_cache_gb=gb)
    with pytest.raises(AssertionError, match='device work'):
        ContinuousGenerator(m, slots=4, kv_cache_gb=gb, kv_cache_dtype='fp8')


def test_generator_passes_the_fp8_page_count(monkeypatch):
    seen = {}

    def fake_init(self, lm, slots, max_gen_len, max_text, **kw):
        seen.update(kw)
        raise AssertionError('device work')

    monkeypatch.setattr(SlotSession, '__init__', fake_init)
    m = _fake_model()
    with pytest.raises(AssertionError):
        ContinuousGenerator(m, slots=8, kv_cache_gb=1.0, kv_cache_dtype='fp8')
    assert seen['kv_pages'] == kv_pages_for_budget(m.lm, 1.0, 'fp8') and seen['kv_dtype'] == 'fp8'
    with pytest.raises(AssertionError):
        ContinuousGenerator(m, slots=8, kv_cache_gb=1.0)
    assert seen['kv_pages'] == kv_pages_for_budget(m.lm, 1.0) and seen['kv_dtype'] == 'fp16'


def test_header_declares_the_fp8_entry_point():
    import os
    from tests import helpers as H
    header = open(os.path.join(H.ROOT, 'include', 'audiocraft_b200.h')).read()
    assert 'acb_lm_begin_slots_paged_fp8' in _lib.EXPORTS and 'int acb_lm_begin_slots_paged_fp8(' in header
