"""GPU parity: EnCodec kernels (through the C-ABI) vs the CPU oracle and the committed reference golden vectors.
Tolerances: RVQ indices bit-exact on identical latents (mismatches tolerated only where the oracle's own
best-vs-second score gap is below fp32 noise, reported); fp32 activations atol 1e-4 (fp32 FMA, different
summation order than the CPU convs)."""
import os

import pytest
import torch

from tests import helpers as H
from audiocraft_b200 import synth
from oracle import encodec_oracle as EO

pytestmark = pytest.mark.gpu


def _lib():
    from audiocraft_b200 import _lib
    return _lib, _lib.lib()


def _dev(t):
    return t.cuda().contiguous()


@pytest.mark.parametrize('cin,cout,k,s,d,causal,L', [
    (1, 64, 7, 1, 1, False, 500), (64, 32, 3, 1, 1, False, 333), (32, 64, 1, 1, 1, False, 333),
    (64, 128, 8, 4, 1, False, 1001), (16, 8, 3, 1, 2, False, 77), (8, 16, 10, 5, 1, False, 203),
    (8, 16, 16, 8, 1, True, 130), (4, 3, 7, 1, 1, True, 50), (4, 2, 7, 1, 1, False, 3), (4, 2, 3, 1, 4, False, 2),
    (24, 1, 7, 1, 1, False, 1000), (3, 5, 4, 2, 1, True, 1), (130, 70, 3, 1, 1, False, 140),
])
def test_conv1d_matches_oracle(cin, cout, k, s, d, causal, L):
    from audiocraft_b200.encodec import conv_geometry
    lib, L_ = _lib()
    g = torch.Generator().manual_seed(cin * 1000 + cout + k + L)
    x = torch.randn(2, cin, L, generator=g)
    w = torch.randn(cout, cin, k, generator=g) / (cin * k) ** 0.5
    b = torch.randn(cout, generator=g)
    for elu, with_res, prec in [(False, False, 0), (True, True, 0), (True, True, 1), (False, False, 1), (True, True, 2)]:
        ref = EO.sconv1d(EO.elu(x) if elu else x, w, b, stride=s, dilation=d, causal=causal)
        res = torch.randn(ref.shape, generator=g) if with_res else None
        if with_res:
            ref = ref + res
        left, tv, tout = conv_geometry(L, k, s, d, causal, True)
        assert tout == ref.shape[-1]
        xd, wd, bd = _dev(x), _dev(w.permute(1, 2, 0).reshape(cin * k, cout)), _dev(b)
        rd = _dev(res) if with_res else None
        y = torch.empty(2, cout, tout, device='cuda')
        lib.check(L_.acb_conv1d(lib.ptr(xd), lib.ptr(wd), lib.ptr(bd), lib.ptr(rd), lib.ptr(y), 2, cin, cout, L, tv, tout,
                                k, s, d, left, 1, int(elu), prec, lib.stream()))
        # prec 1 = 3xTF32 on the tensor pipe (fp32 FMA fallback for tiny layers): same tolerance, one layer deep
        torch.testing.assert_close(y.cpu(), ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('cin,cout,k,s,d,causal,L', [
    (64, 128, 8, 4, 1, False, 1001), (128, 64, 3, 1, 1, False, 333), (8, 64, 7, 1, 1, False, 500), (16, 128, 10, 5, 1, False, 2003),
    (64, 256, 16, 8, 1, True, 4100), (8, 64, 3, 1, 2, False, 77), (8, 64, 7, 1, 1, False, 3), (512, 1024, 16, 8, 1, False, 4000),
])
def test_experimental_conv1d_t6_matches_oracle(cin, cout, k, s, d, causal, L):
    """Implicit-GEMM wgmma convolution with per-8-channel fp32 flushes of the tensor-core accumulator (acb_conv1d_t6): same
    contract as acb_conv1d; the flush is meant to bring the tensor-core path to fp32-FMA accuracy (atol 2e-5 here, vs 1e-4
    for the un-flushed 3xTF32 kernels one layer deep)."""
    from audiocraft_b200.encodec import conv_geometry, pack_conv_t6
    lib, L_ = _lib()
    g = torch.Generator().manual_seed(cin * 1000 + cout + k + L)
    x = torch.randn(2, cin, L, generator=g)
    w = torch.randn(cout, cin, k, generator=g) / (cin * k) ** 0.5
    b = torch.randn(cout, generator=g)
    tile = L_.acb_conv1d_t6_tile(cout)
    assert tile in (64, 128)
    w6 = _dev(pack_conv_t6(w, tile))
    for elu, with_res in [(False, False), (True, True)]:
        ref = EO.sconv1d(EO.elu(x) if elu else x, w, b, stride=s, dilation=d, causal=causal)
        res = torch.randn(ref.shape, generator=g) if with_res else None
        if with_res:
            ref = ref + res
        left, tv, tout = conv_geometry(L, k, s, d, causal, True)
        xd, bd = _dev(x), _dev(b)
        rd = _dev(res) if with_res else None
        y = torch.full((2, cout, tout), float('nan'), device='cuda')
        lib.check(L_.acb_conv1d_t6(lib.ptr(xd), lib.ptr(w6), lib.ptr(bd), lib.ptr(rd), lib.ptr(y), 2, cin, cout, L, tv, tout,
                                   k, s, d, left, 1, int(elu), lib.stream()))
        torch.cuda.synchronize()
        print(f'conv1d_t6 {cin}->{cout} k{k} s{s}: max err {(y.cpu() - ref).abs().max():.2e}')
        torch.testing.assert_close(y.cpu(), ref, rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize('C,d,causal,L,B', [(64, 1, False, 1000, 2), (64, 1, False, 128, 1), (128, 1, False, 333, 3), (256, 1, False, 257, 2),
                                           (64, 2, False, 517, 2), (128, 1, True, 130, 2), (64, 1, False, 3, 1), (256, 3, True, 1025, 1)])
@pytest.mark.parametrize('split', ['fp16x2', 'tf32x3'])
def test_resblock_matches_oracle(monkeypatch, split, C, d, causal, L, B):
    """SEANetResnetBlock with the identity skip as one kernel (acb_resblock; seanet.py:44-69): y = x + conv1x1(elu(conv3(elu(x)))).
    exact = 1 (the encoder setting, tensor-core runs cut every 24 / 16 reduction rows) to 2e-5, exact = 0 (3xTF32 straight) to 1e-4 --
    the tolerances of the flushed / un-flushed single-layer kernels."""
    from audiocraft_b200.encodec import conv_geometry
    lib, L_ = _lib()
    if split == 'tf32x3':      # the round-2 first version of the kernel (operands split into tf32 terms); default: fp16 terms
        monkeypatch.setenv('ACB_RESBLOCK_TF32', '1')
    assert L_.acb_resblock_supported(C, 3, d) == 1 and L_.acb_resblock_supported(512, 3, 1) == 0
    g = torch.Generator().manual_seed(C * 100 + d * 10 + L)
    x = torch.randn(B, C, L, generator=g)
    w1 = torch.randn(C // 2, C, 3, generator=g) / (3 * C) ** 0.5
    b1 = torch.randn(C // 2, generator=g) * 0.3
    w2 = torch.randn(C, C // 2, 1, generator=g) / (C // 2) ** 0.5
    b2 = torch.randn(C, generator=g) * 0.3
    hid = EO.sconv1d(EO.elu(x), w1, b1, stride=1, dilation=d, causal=causal)
    ref = x + EO.sconv1d(EO.elu(hid), w2, b2, stride=1, dilation=1, causal=causal)
    left, tv, tout = conv_geometry(L, 3, 1, d, causal, True)
    assert tout == L and tv == L
    xd, b1d, b2d = _dev(x), _dev(b1), _dev(b2)
    w1d = _dev(w1.permute(2, 1, 0))                 # [k][C][C/2]
    w2d = _dev(w2[:, :, 0].t())                     # [C/2][C]
    for exact, tol in ((1, 2e-5), (0, 1e-4)):
        y = torch.full((B, C, L), float('nan'), device='cuda')
        lib.check(L_.acb_resblock(lib.ptr(xd), lib.ptr(w1d), lib.ptr(b1d), lib.ptr(w2d), lib.ptr(b2d), lib.ptr(y), B, C, L, 3, d,
                                  left, 1, exact, lib.stream()))
        torch.cuda.synchronize()
        print(f'resblock[{split}] C={C} dil={d} L={L} exact={exact}: max err {(y.cpu() - ref).abs().max():.2e}')
        torch.testing.assert_close(y.cpu(), ref, rtol=tol, atol=tol)


@pytest.mark.parametrize('cin,cout,s,causal,ratio,L', [
    (16, 8, 2, False, 1.0, 37), (8, 16, 3, True, 1.0, 20), (32, 16, 4, False, 1.0, 101), (12, 6, 5, False, 1.0, 50),
    (64, 32, 8, False, 1.0, 50), (8, 4, 4, True, 0.5, 33), (8, 4, 8, True, 0.0, 1), (70, 66, 4, False, 1.0, 70),
    (128, 64, 4, False, 1.0, 300), (96, 40, 5, False, 1.0, 131), (64, 16, 8, True, 1.0, 257), (256, 128, 2, True, 0.5, 129),
])
def test_convtr1d_matches_oracle(cin, cout, s, causal, ratio, L):
    from audiocraft_b200.encodec import convtr_geometry
    lib, L_ = _lib()
    g = torch.Generator().manual_seed(cin + cout + s + L)
    x = torch.randn(2, cin, L, generator=g)
    w = torch.randn(cin, cout, 2 * s, generator=g) / (2 * cin) ** 0.5
    b = torch.randn(cout, generator=g)
    ref = EO.sconvtr1d(EO.elu(x), w, b, s, causal, ratio)
    tl, tout = convtr_geometry(L, 2 * s, s, causal, ratio)
    assert tout == ref.shape[-1] == L * s
    xd, wd, bd = _dev(x), _dev(w.permute(0, 2, 1)), _dev(b)   # keep the device tensors alive across the launch
    wg = _dev(w.view(cin, cout, 2, s).flip(2).permute(0, 2, 1, 3).reshape(cin * 2, cout * s))
    for prec in (0, 1):   # fp32 FMA; 3xTF32 on wgmma as one GEMM over virtual channels (when the layer is big enough)
        y = torch.empty(2, cout, tout, device='cuda')
        lib.check(L_.acb_convtr1d(lib.ptr(xd), lib.ptr(wd), lib.ptr(wg), lib.ptr(bd), lib.ptr(y), 2, cin,
                                  cout, L, tout, 2 * s, s, tl, 1, prec, lib.stream()))
        torch.testing.assert_close(y.cpu(), ref, rtol=1e-4, atol=1e-4)


def test_weight_norm_fold_matches_oracle():
    lib, L_ = _lib()
    g = torch.Generator().manual_seed(0)
    for shape in [(64, 32, 3), (5, 1, 7), (128, 64, 16)]:
        v = torch.randn(shape, generator=g)
        gg = torch.rand(shape[0], 1, 1, generator=g) + 0.5
        w = torch.empty(shape, device='cuda')
        vd, gd = _dev(v), _dev(gg)
        lib.check(L_.acb_weight_norm_fold(lib.ptr(vd), lib.ptr(gd), lib.ptr(w), shape[0], shape[1] * shape[2],
                                          lib.stream()))
        torch.testing.assert_close(w.cpu(), EO.fold_weight_norm(gg, v), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('hidden,batch,T,layers', [(64, 3, 20, 2), (512, 2, 9, 1), (1024, 9, 6, 2), (8, 1, 1, 1)])
def test_lstm_matches_oracle(hidden, batch, T, layers):
    from audiocraft_b200.encodec import EncodecModel
    g = torch.Generator().manual_seed(hidden + T)
    sd = {}
    bnd = 1.0 / hidden ** 0.5
    for n in range(layers):
        for nm, shp in [('weight_ih', (4 * hidden, hidden)), ('weight_hh', (4 * hidden, hidden)), ('bias_ih', (4 * hidden,)),
                        ('bias_hh', (4 * hidden,))]:
            sd[f'l.{nm}_l{n}'] = (torch.rand(shp, generator=g) * 2 - 1) * bnd
    x = torch.randn(batch, hidden, T, generator=g)
    ref = EO.lstm_block(x, sd, 'l.', layers)
    m = EncodecModel.__new__(EncodecModel)  # only the LSTM launcher is exercised
    from audiocraft_b200 import _lib
    m._lib, m.device, m.launches, m._lstm_prec = _lib.lib(), torch.device('cuda'), 0, 0
    layer = m._prepare(dict(kind='lstm', prefix='l.', dim=hidden, layers=layers), sd)
    y = m._lstm(_dev(x), layer)
    torch.testing.assert_close(y.cpu(), ref, rtol=1e-4, atol=2e-5)


def _codes_match(codes_gpu, codes_ref, margins, what):
    """Bit-exact, except where the oracle's own top-2 gap is below fp32 summation noise (reported)."""
    neq = codes_gpu != codes_ref
    if neq.any():
        # a flipped code changes every later residual: only judge the FIRST differing codebook of each frame
        first = neq.int().cumsum(1).eq(1) & neq
        gaps = margins[first]
        print(f"{what}: {int(first.sum())} near-tie code flips, oracle margins {gaps.tolist()[:8]}")
        assert (gaps.abs() < 1e-4).all(), f"{what}: RVQ index mismatch with a clear margin"


@pytest.mark.parametrize('B,D,T,nq,bins', [(2, 128, 333, 4, 2048), (1, 32, 31, 4, 64), (3, 128, 1, 8, 1024), (1, 128, 4000, 4, 2048)])
def test_rvq_encode_decode_match_oracle(B, D, T, nq, bins):
    lib, L_ = _lib()
    g = torch.Generator().manual_seed(B * D + T)
    z = torch.randn(B, D, T, generator=g) * 0.4
    cbs = [torch.randn(bins, D, generator=g) * 0.35 * 0.6 ** k for k in range(nq)]
    ref, margins = EO.rvq_encode(z, cbs, return_margin=True)
    cb = _dev(torch.stack(cbs))
    codes = torch.empty(B, nq, T, dtype=torch.int64, device='cuda')
    zd, cbn = _dev(z), cb.pow(2).sum(-1).contiguous()
    lib.check(L_.acb_rvq_encode(lib.ptr(zd), lib.ptr(cb), lib.ptr(cbn), lib.ptr(codes), B, D, T,
                                nq, bins, lib.stream()))
    _codes_match(codes.cpu(), ref, margins, 'rvq_encode')
    out = torch.empty(B, D, T, device='cuda')
    refd = _dev(ref)
    lib.check(L_.acb_rvq_decode(lib.ptr(refd), lib.ptr(cb), lib.ptr(out), B, D, T, nq, bins, lib.stream()))
    torch.testing.assert_close(out.cpu(), EO.rvq_decode(ref, cbs), rtol=0, atol=1e-6)


@pytest.mark.parametrize('name', ['encodec_tiny', 'encodec_tiny_causal', 'encodec_24k', 'encodec_32k'])
def test_encodec_model_matches_reference_golden(name):
    """End to end against the REAL reference's outputs (tests/golden, generated by tests/golden/make_golden.py)."""
    from audiocraft_b200.encodec import EncodecModel
    g = torch.load(os.path.join(H.GOLDEN_DIR, f'{name}.pt'), weights_only=False)
    cfg = synth.ENCODEC_CONFIGS[name]
    sd = synth.synth_encodec_state_dict(cfg, seed=g['wseed'])
    x = H.audio_input(cfg, g['batch'], g['length'], g['xseed'])
    m = EncodecModel(sd, cfg)   # defaults: fp32 encoder (index-exact), 3xTF32 decoder
    lat = m.encode_latent(m.preprocess(x.cuda())[0])
    torch.testing.assert_close(lat.cpu(), g['latent'], rtol=0, atol=1e-4)
    codes, scale = m.encode(x)
    assert codes.dtype == torch.int64 and codes.shape == g['codes'].shape
    # margins from the oracle on the golden latent
    _, margins = EO.rvq_encode(g['latent'], EO.codebooks_of(sd, cfg['n_q']), return_margin=True)
    _codes_match(codes.cpu(), g['codes'], margins, name)
    if g['scale'] is not None:
        torch.testing.assert_close(scale.cpu(), g['scale'], rtol=1e-5, atol=0)
    sc = None if g['scale'] is None else g['scale'].cuda()
    for mdl, tol in ((m, 1e-4), (EncodecModel(sd, cfg, decoder_precision='fp32'), 2e-5)):
        wav = mdl.decode(g['codes'].cuda(), sc).cpu()
        if 'wav' in g:
            print(f'{name} decoder max err {(wav - g["wav"]).abs().max():.2e} (tol {tol})')
            torch.testing.assert_close(wav, g['wav'], rtol=0, atol=tol)
        else:
            assert wav.shape[-1] == g['wav_len']
            print(f'{name} decoder max err {(wav[..., ::g["wav_stride"]] - g["wav_strided"]).abs().max():.2e} (tol {tol})')
            torch.testing.assert_close(wav[..., :512], g['wav_head'], rtol=0, atol=tol)
            torch.testing.assert_close(wav[..., ::g['wav_stride']], g['wav_strided'], rtol=0, atol=tol)


def test_encodec_32k_properties_at_size():
    """Size-independent properties at a bench-like size: length round trip (reference test_encodec_model.py:37-46),
    batch independence, determinism, and oracle agreement on a slice."""
    from audiocraft_b200.encodec import EncodecModel
    cfg = synth.ENCODEC_CONFIGS['encodec_32k']
    sd = synth.synth_encodec_state_dict(cfg, seed=0)
    m = EncodecModel(sd, cfg)
    x = H.audio_input(cfg, 6, 64000 + 123, 3)
    codes, scale = m.encode(x)
    assert scale is None and codes.shape == (6, 4, -(-x.shape[-1] // 640))
    assert int(codes.min()) >= 0 and int(codes.max()) < 2048
    wav = m.decode(codes)
    assert wav.shape == (6, 1, codes.shape[-1] * 640) and wav.shape[-1] >= x.shape[-1]
    assert torch.isfinite(wav).all()
    codes2, _ = m.encode(x)
    assert torch.equal(codes, codes2) and torch.equal(wav, m.decode(codes))      # deterministic
    c1, _ = m.encode(x[2:3])
    assert torch.equal(c1, codes[2:3])                                           # items are independent
    torch.testing.assert_close(m.decode(codes[4:5]), wav[4:5], rtol=0, atol=1e-6)
    o = EO.EncodecOracle(sd, cfg)
    oc, _ = o.encode(x[:1, :, :16000])
    gc, _ = m.encode(x[:1, :, :16000])
    lat = o.encode_latent(x[:1, :, :16000])
    _, margins = EO.rvq_encode(lat, EO.codebooks_of(sd, 4), return_margin=True)
    _codes_match(gc.cpu(), oc, margins, 'encodec_32k slice')
    torch.testing.assert_close(m.decode(oc.cuda()).cpu(), o.decode(oc), rtol=0, atol=1e-4)


def test_set_num_codebooks_and_errors():
    from audiocraft_b200.encodec import EncodecModel
    cfg = synth.ENCODEC_CONFIGS['encodec_tiny']
    m = EncodecModel(synth.synth_encodec_state_dict(cfg, 1), cfg)
    x = H.audio_input(cfg, 1, 400, 1)
    full, _ = m.encode(x)
    m.set_num_codebooks(2)
    part, _ = m.encode(x)
    assert part.shape[1] == 2 and torch.equal(part, full[:, :2]) and m.num_codebooks == 2 and m.total_codebooks == 4
    assert m.decode(part).shape == m.decode(full).shape
    with pytest.raises(AssertionError):
        m.set_num_codebooks(5)
    with pytest.raises(AssertionError):
        m.encode(torch.zeros(1, 3, 100))


def test_interleave_stereo_wrapper_matches_reference_golden():
    """SURVEY section 8f.1: stereo MusicGen's codec wrapper (audiocraft/models/encodec.py:393-506)."""
    from audiocraft_b200.encodec import EncodecModel, InterleaveStereoCompressionModel
    g = torch.load(os.path.join(H.GOLDEN_DIR, 'encodec_tiny_stereo.pt'), weights_only=False)
    cfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'])
    cfg['renormalize'] = False
    mono = EncodecModel(synth.synth_encodec_state_dict(cfg, seed=g['wseed']), cfg)
    cfg2 = dict(cfg)
    cfg2['channels'] = 2
    x = H.audio_input(cfg2, g['batch'], g['length'], g['xseed'])
    for pt in (False, True):
        w = InterleaveStereoCompressionModel(mono, per_timestep=pt)
        assert (w.num_codebooks, w.frame_rate, w.channels, w.cardinality, w.total_codebooks) == g[f'props_pt{int(pt)}']
        codes, scale = w.encode(x.cuda())
        assert scale is None and torch.equal(codes.cpu(), g[f'codes_pt{int(pt)}'])
        wav = w.decode(g[f'codes_pt{int(pt)}'].cuda())
        torch.testing.assert_close(wav.cpu(), g[f'wav_pt{int(pt)}'], rtol=0, atol=1e-4)
        l, r = w.get_left_right_codes(codes)
        c0, _ = mono.encode(x[:, :1].cuda())
        assert torch.equal(l, c0)
    with pytest.raises(AssertionError):
        InterleaveStereoCompressionModel(mono).encode(x[:, :1].cuda())


@pytest.mark.parametrize('name', ['encodec_24k', 'encodec_32k'])
def test_tensor_core_encoder_mode(name):
    """encoder_precision='tf32x3' (throughput mode): latents within 5e-4 of the fp32 reference (tensor-core accumulate
    rounding grows through 15 layers + LSTM), codes equal wherever the oracle's margin is clear of that."""
    from audiocraft_b200.encodec import EncodecModel
    g = torch.load(os.path.join(H.GOLDEN_DIR, f'{name}.pt'), weights_only=False)
    cfg = synth.ENCODEC_CONFIGS[name]
    sd = synth.synth_encodec_state_dict(cfg, seed=g['wseed'])
    x = H.audio_input(cfg, g['batch'], g['length'], g['xseed'])
    m = EncodecModel(sd, cfg, encoder_precision='tf32x3')
    lat = m.encode_latent(x.cuda()).cpu()
    print(f'{name} tensor-core encoder latent max err {(lat - g["latent"]).abs().max():.2e}')
    torch.testing.assert_close(lat, g['latent'], rtol=0, atol=5e-4)
    codes, _ = m.encode(x)
    _, margins = EO.rvq_encode(g['latent'], EO.codebooks_of(sd, cfg['n_q']), return_margin=True)
    neq = codes.cpu() != g['codes']
    first = neq.int().cumsum(1).eq(1) & neq
    assert (margins[first].abs() < 5e-3).all()
    assert (codes.cpu() == g['codes']).float().mean() > 0.98


@pytest.mark.parametrize('name', ['encodec_32k', 'encodec_24k'])
def test_experimental_flush_encoder_mode(name):
    """encoder_precision='tf32x3_flush': the implicit-GEMM wgmma convs with per-8-channel fp32 flushes are meant to make
    the tensor-core encoder as accurate as the fp32 FMA one (latents atol 2e-5, codes under the exact-encoder rule)."""
    from audiocraft_b200.encodec import EncodecModel
    g = torch.load(os.path.join(H.GOLDEN_DIR, f'{name}.pt'), weights_only=False)
    cfg = synth.ENCODEC_CONFIGS[name]
    sd = synth.synth_encodec_state_dict(cfg, seed=g['wseed'])
    x = H.audio_input(cfg, g['batch'], g['length'], g['xseed'])
    m = EncodecModel(sd, cfg, encoder_precision='tf32x3_flush')
    lat = m.encode_latent(x.cuda()).cpu()
    print(f'{name} flush-mode encoder latent max err {(lat - g["latent"]).abs().max():.2e}')
    torch.testing.assert_close(lat, g['latent'], rtol=0, atol=2e-5)
    codes, _ = m.encode(x)
    assert (codes.cpu() == g['codes']).float().mean() > 0.999


@pytest.mark.parametrize('shortcut', [False, True])
def test_hf_encodec_checkpoint_on_kernels(shortcut):
    """SURVEY section 8f.1: an HF-format EnCodec checkpoint (random init here) converted and run on the kernels vs
    transformers' own CPU implementation; exercises the conv-shortcut residual block and n_q = 32."""
    import warnings
    from transformers import EncodecConfig, EncodecModel as HFModel
    from audiocraft_b200.encodec import HFEncodecCompressionModel, hf_encodec_to_reference
    warnings.filterwarnings('ignore')
    hc = EncodecConfig(use_conv_shortcut=shortcut)
    torch.manual_seed(0)
    hf = HFModel(hc).eval()
    hsd = hf.state_dict()
    g = torch.Generator().manual_seed(1)
    for k in hsd:
        if k.endswith('codebook.embed'):
            hsd[k].copy_(torch.randn(hsd[k].shape, generator=g) * 0.5)
    x = torch.randn(2, 1, 5000, generator=g) * 0.3
    with torch.no_grad():
        enc = hf.encode(x, None, 24.0)
        dec = hf.decode(enc[0], enc[1])[0]
    m = HFEncodecCompressionModel(hsd, hc)
    assert m.sample_rate == 24000 and m.cardinality == 1024 and m.num_codebooks == 32 and m.total_codebooks == 32
    codes, scale = m.encode(x)
    sd, cfg = hf_encodec_to_reference(hsd, hc)
    lat = EO.EncodecOracle(sd, cfg).encode_latent(x)
    _, margins = EO.rvq_encode(lat, EO.codebooks_of(sd, 32), return_margin=True)
    _codes_match(codes.cpu(), enc[0][0], margins, f'hf encodec shortcut={shortcut}')
    torch.testing.assert_close(m.decode(enc[0][0].cuda()).cpu(), dec, rtol=0, atol=1e-4)
    m.set_num_codebooks(8)
    c8, _ = m.encode(x)
    assert c8.shape[1] == 8
    with pytest.raises(ValueError):
        m.set_num_codebooks(5)
