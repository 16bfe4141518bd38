"""EnCodec 48 kHz on the GPU: the GroupNorm statistics / apply and overlap-add kernels against float64 on their own inputs, the
GroupNorm codec end to end against transformers' 48 kHz model and the reference's own GroupNorm EncodecModel (golden), and
the reference wrapper's one-chunk contract."""
import os

import pytest
import torch

from audiocraft_b200 import synth
from oracle import encodec_oracle as EO
from tests import encodec_gn_oracle as GO
from tests import helpers as H
from tests.test_gpu_encodec import _codes_match

pytestmark = pytest.mark.gpu


def _lib():
    from audiocraft_b200 import _lib
    return _lib, _lib.lib()


def _stats(x, eps=1e-5):
    lib, L = _lib()
    B, C, T = x.shape
    ws = torch.empty(int(L.acb_groupnorm_workspace_bytes(B, C, T)), dtype=torch.uint8, device='cuda')
    st = torch.empty(B, 2, dtype=torch.float64, device='cuda')
    lib.check(L.acb_groupnorm_stats(lib.ptr(x), lib.ptr(ws), lib.ptr(st), B, C, T, eps, lib.stream()))
    return st


def _apply(x, st, g, b, left=0, t_out=None, x2=None, st2=None, g2=None, b2=None, res=None):
    lib, L = _lib()
    B, C, T = x.shape
    t_out = T if t_out is None else t_out
    y = torch.empty(B, C, t_out, device='cuda')
    lib.check(L.acb_groupnorm_apply(lib.ptr(x), lib.ptr(st), lib.ptr(g), lib.ptr(b), T, left, lib.ptr(x2), lib.ptr(st2), lib.ptr(g2),
                                    lib.ptr(b2), lib.ptr(res), lib.ptr(y), B, C, t_out, lib.stream()))
    return y


def _gn64(x, g, b, eps=1e-5):
    x = x.double().cpu()
    m = x.mean(dim=(1, 2), keepdim=True)
    v = (x - m).pow(2).mean(dim=(1, 2), keepdim=True)
    return (x - m) / (v + eps).sqrt() * g.double().cpu().view(1, -1, 1) + b.double().cpu().view(1, -1, 1), m.view(-1), v.view(-1)


def _affine(C, seed):
    g = torch.Generator().manual_seed(seed)
    return (1 + 0.3 * torch.randn(C, generator=g)).cuda(), (0.2 * torch.randn(C, generator=g)).cuda()


@pytest.mark.parametrize('C,T,B', [(2, 48001, 3), (16, 6001, 2), (32, 47999, 2), (512, 1203, 2), (1024, 6000 - 7, 1)])
def test_groupnorm_stats_and_apply_match_float64(C, T, B):
    g = torch.Generator().manual_seed(C + T)
    x = (torch.randn(B, C, T, generator=g) * 2 + 0.5).cuda()
    gam, bet = _affine(C, C)
    st = _stats(x)
    ref, m, v = _gn64(x, gam, bet)
    torch.testing.assert_close(st[:, 0].cpu(), m, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(st[:, 1].cpu(), 1 / (v + 1e-5).sqrt(), rtol=1e-10, atol=0)
    y = _apply(x, st, gam, bet)
    torch.testing.assert_close(y.cpu().double(), ref, rtol=0, atol=5e-6)
    # the end of a residual block: GN(shortcut) + GN(conv2), and GN(conv2) + the identity skip
    x2 = (torch.randn(B, C, T, generator=g) - 3).cuda()
    g2, b2 = _affine(C, C + 1)
    ref2 = _gn64(x2, g2, b2)[0]
    y = _apply(x, st, gam, bet, x2=x2, st2=_stats(x2), g2=g2, b2=b2)
    torch.testing.assert_close(y.cpu().double(), ref + ref2, rtol=0, atol=1e-5)
    y = _apply(x, st, gam, bet, res=x2)
    torch.testing.assert_close(y.cpu().double(), ref + x2.cpu().double(), rtol=0, atol=1e-5)


def test_groupnorm_large_mean_small_spread():
    """mean 1e3, std 1e-2: an fp32 E[x^2] - E[x]^2 loses the variance entirely; the kernel's output stays within 1e-5."""
    g = torch.Generator().manual_seed(5)
    x = (1e3 + 1e-2 * torch.randn(2, 32, 20011, generator=g)).cuda()
    x32 = x.cpu()
    naive = (x32.pow(2).mean(dim=(1, 2)) - x32.mean(dim=(1, 2)).pow(2))
    gam, bet = _affine(32, 6)
    ref, m, v = _gn64(x, gam, bet)
    assert ((naive.double() - v).abs() / v).max() > 1e-2        # the float32 one-pass variance fails here
    y = _apply(x, _stats(x), gam, bet).cpu().double()
    assert ((y - ref).abs() / ref.abs().clamp_min(1)).max() < 1e-5


def test_groupnorm_constant_input():
    x = torch.full((2, 16, 1001), 0.75, device='cuda')
    st = _stats(x).cpu()
    assert torch.equal(st[:, 0], torch.full((2,), 0.75, dtype=torch.float64))
    eps = torch.tensor(1e-5, dtype=torch.float32).item()           # the kernel takes eps as a float
    torch.testing.assert_close(st[:, 1], torch.full((2,), 1 / eps ** 0.5, dtype=torch.float64), rtol=1e-12, atol=0)
    gam, bet = _affine(16, 3)
    torch.testing.assert_close(_apply(x, _stats(x), gam, bet).cpu(), bet.cpu().view(1, -1, 1).expand(2, 16, 1001), rtol=0, atol=0)


def test_groupnorm_item_independent_of_batch():
    g = torch.Generator().manual_seed(9)
    x = torch.randn(40, 32, 48000 // 8 + 3, generator=g).cuda()
    gam, bet = _affine(32, 1)
    st = _stats(x)
    y = _apply(x, st, gam, bet)
    for i in (0, 17, 39):
        one = x[i:i + 1].contiguous()
        assert torch.equal(_stats(one), st[i:i + 1])
        assert torch.equal(_apply(one, _stats(one), gam, bet), y[i:i + 1])


def test_groupnorm_transposed_conv_window():
    """NormConvTranspose1d normalises the FULL transposed-conv output and the trim comes after: statistics of the trimmed
    window are a different (wrong) answer."""
    lib, L = _lib()
    g = torch.Generator().manual_seed(2)
    B, cin, cout, S, T = 2, 64, 32, 8, 37
    x = torch.randn(B, cin, T, generator=g)
    w = torch.randn(cin, cout, 2 * S, generator=g) / cin ** 0.5
    bias = torch.randn(cout, generator=g) * 3    # large bias at the edges makes the trimmed steps matter
    full = torch.nn.functional.conv_transpose1d(x.double(), w.double(), bias.double(), stride=S)
    y_full = torch.empty(B, cout, (T + 1) * S, device='cuda')
    xd, wd, bd = x.cuda(), w.permute(0, 2, 1).contiguous().cuda(), bias.cuda()     # [Cin][K][Cout]
    lib.check(L.acb_convtr1d(lib.ptr(xd), lib.ptr(wd), None, lib.ptr(bd), lib.ptr(y_full), B, cin, cout, T, (T + 1) * S, 2 * S, S,
                             0, 0, 0, lib.stream()))
    torch.testing.assert_close(y_full.cpu().double(), full, rtol=0, atol=1e-4)
    gam, bet = _affine(cout, 4)
    left, right = S - S // 2, S // 2
    ref = _gn64(full, gam, bet)[0][..., left:full.shape[-1] - right]
    y = _apply(y_full, _stats(y_full), gam, bet, left=left, t_out=T * S)
    torch.testing.assert_close(y.cpu().double(), ref, rtol=0, atol=1e-5)
    trimmed = y_full[..., left:left + T * S].contiguous()
    wrong = _apply(trimmed, _stats(trimmed), gam, bet).cpu().double()
    assert (wrong - ref).abs().max() > 1e-3


@pytest.mark.parametrize('n,t_last,scaled', [(1, 1440, True), (2, 48000, False), (2, 1600, True), (11, 4800, True)])
def test_overlap_add_matches_float64(n, t_last, scaled):
    lib, L = _lib()
    g = torch.Generator().manual_seed(n)
    B, C, tf, stride = 2, 2, 48000, 47520
    frames = [torch.randn(B, C, tf, generator=g) for _ in range(n - 1)] + [torch.randn(B, C, t_last, generator=g)]
    if n == 1:
        frames = [frames[-1]]
    scales = [torch.rand(B, 1, generator=g) + 0.5 for _ in range(n)]
    ref = GO.linear_overlap_add([(f * s.view(-1, 1, 1) if scaled else f).double() for f, s in zip(frames, scales)], stride)
    t_total = stride * (n - 1) + t_last
    y = torch.empty(B, C, t_total, device='cuda')
    full = torch.stack(frames[:-1]).cuda().contiguous() if n > 1 else None
    sc = torch.stack([s.view(-1) for s in scales]).cuda() if scaled else None
    last = frames[-1].cuda()
    lib.check(L.acb_overlap_add(lib.ptr(full), lib.ptr(last), lib.ptr(sc), lib.ptr(y), n, B, C, tf if n > 1 else t_last,
                                t_last, stride, t_total, lib.stream()))
    torch.testing.assert_close(y.cpu().double(), ref, rtol=0, atol=2e-6)


# ----------------------------------------------------------------------------- end to end against transformers

_HF = {}


def _models():
    if not _HF:
        from audiocraft_b200.encodec import HFEncodecCompressionModel
        hf = GO.hf_48k_model(seed=0)
        _HF['hf'], _HF['m'] = hf, HFEncodecCompressionModel(hf.state_dict(), hf.config)
    return _HF['hf'], _HF['m']


def _margins(hf, x, scales, sd):
    """Per chunk, the oracle's best-vs-second RVQ score gap on transformers' own latent."""
    out = []
    for i, o in enumerate(range(0, x.shape[-1], 47520)):
        with torch.no_grad():
            lat = hf.encoder(x[..., o:o + 48000] / scales[i].view(-1, 1, 1))
        m = EO.rvq_encode(lat, EO.codebooks_of(sd, 16), return_margin=True)[1]
        out.append(m)
    F = out[0].shape[-1]
    out[-1] = torch.nn.functional.pad(out[-1], (0, F - out[-1].shape[-1]), value=1.0)
    return torch.stack(out)


@pytest.mark.parametrize('seconds,B', [(0.9, 1), (0.9, 2), (3.0, 1), (3.0, 2), (10.0, 2)])
def test_encodec48_matches_transformers(seconds, B):
    from audiocraft_b200.encodec import hf_encodec_to_reference
    hf, m = _models()
    sd, _ = hf_encodec_to_reference(hf.state_dict(), hf.config)
    x = H.audio_input(dict(sample_rate=48000, channels=2), B, int(seconds * 48000), 7)
    x[-1] *= 4.0                                   # items of different loudness: per-item, per-chunk scales
    with torch.no_grad():
        r_codes, r_scales, r_pad = hf.encode(x, None, 24.0, return_dict=False)
    margins = _margins(hf, x, r_scales, sd)
    for bw, nq in zip([3.0, 6.0, 12.0, 24.0], [2, 4, 8, 16]):
        codes, scales, pad = m.model.encode(x, None, bw)
        F = r_codes.shape[-1]
        assert codes.shape == (r_codes.shape[0], B, nq, F) and pad == r_pad and len(scales) == len(r_scales)
        for a, b in zip(scales, r_scales):
            torch.testing.assert_close(a.cpu(), b, rtol=1e-6, atol=0)
        for i in range(codes.shape[0]):
            n = F - (pad if i == codes.shape[0] - 1 else 0)
            _codes_match(codes[i, ..., :n].cpu(), r_codes[i, :, :nq, :n], margins[i, :, :nq, :n], f'48k {seconds}s B={B} bw={bw}')
        ref_codes = r_codes[:, :, :nq]
        with torch.no_grad():
            ref = hf.decode(ref_codes, r_scales, None, False, r_pad)[0]
        wav = m.model.decode(ref_codes.cuda(), [s.cuda() for s in r_scales], None, r_pad)[0].cpu()
        tol = 1e-4 * max(1.0, ref.abs().max().item())
        print(f'48k {seconds}s B={B} bw={bw}: waveform max err {(wav - ref).abs().max():.2e} (tol {tol:.2e})')
        assert wav.shape == ref.shape
        torch.testing.assert_close(wav, ref, rtol=0, atol=tol)
        if codes.shape[0] == 1:                   # the reference wrapper's contract: one chunk, item 0's scale in decode
            m.set_num_codebooks(nq)
            c, s = m.encode(x)
            assert torch.equal(c, codes[0]) and torch.equal(s, scales[0])
            with torch.no_grad():
                ref_w = hf.decode(ref_codes[0][None], r_scales[0], None, False)[0]
            torch.testing.assert_close(m.decode(ref_codes[0].cuda(), r_scales[0].cuda()).cpu(), ref_w, rtol=0,
                                       atol=1e-4 * max(1.0, ref_w.abs().max().item()))
    m.set_num_codebooks(16)


def test_wrapper_one_chunk_contract():
    """HFEncodecCompressionModel.encode fails like the reference's `assert len(res[0]) == 1` on input longer than one chunk,
    and decode applies item 0's scale to every item, as `self.model.decode(codes[None], scale)` does in transformers."""
    hf, m = _models()
    x = H.audio_input(dict(sample_rate=48000, channels=2), 2, 48000 + 1, 1)
    with pytest.raises(AssertionError, match='model.encode'):
        m.encode(x)
    x = x[..., :40000].clone()
    x[1] *= 5.0
    codes, scale = m.encode(x)
    assert scale[1, 0] > 3 * scale[0, 0]
    with torch.no_grad():
        ref = hf.decode(codes.cpu()[None], scale.cpu(), None, False)[0]
    wav = m.decode(codes, scale).cpu()
    torch.testing.assert_close(wav, ref, rtol=0, atol=1e-4 * max(1.0, ref.abs().max().item()))
    unscaled = m.decode(codes).cpu()
    torch.testing.assert_close(wav[1], unscaled[1] * scale[0, 0].item(), rtol=1e-5, atol=1e-6)   # item 1 scaled by item 0's scale
    lat = m.decode_latent(codes)
    with torch.no_grad():
        torch.testing.assert_close(lat.cpu(), hf.quantizer.decode(codes.cpu().transpose(0, 1)), rtol=0, atol=1e-6)


def test_groupnorm_codec_matches_reference_golden():
    """An audiocraft-format GroupNorm codec (the reference's own EncodecModel, norm='time_group_norm') on the kernels."""
    from audiocraft_b200.encodec import EncodecModel
    g = torch.load(os.path.join(H.GOLDEN_DIR, 'encodec_tiny_gn.pt'), weights_only=False)
    cfg = g['cfg']
    sd = synth.synth_encodec_state_dict(cfg, seed=g['wseed'])
    x = H.audio_input(cfg, g['batch'], g['length'], g['xseed'])
    m = EncodecModel(sd, cfg)
    lat = m.encode_latent(m.preprocess(x.cuda())[0]).cpu()
    print(f'gn golden latent max err {(lat - g["latent"]).abs().max():.2e}')
    torch.testing.assert_close(lat, g['latent'], rtol=0, atol=1e-4)
    codes, scale = m.encode(x)
    _, margins = EO.rvq_encode(g['latent'], EO.codebooks_of(sd, cfg['n_q']), return_margin=True)
    _codes_match(codes.cpu(), g['codes'], margins, 'encodec_tiny_gn')
    torch.testing.assert_close(scale.cpu(), g['scale'], rtol=1e-5, atol=0)
    wav = m.decode(g['codes'].cuda(), g['scale'].cuda()).cpu()
    assert wav.shape[-1] == g['wav_len']
    torch.testing.assert_close(wav[..., ::g['wav_stride']], g['wav_strided'], rtol=0, atol=1e-4)


@pytest.mark.parametrize('rate', [24, 48])
def test_get_pretrained_local_transformers_dir(tmp_path, rate):
    from transformers import EncodecConfig, EncodecModel as HFModel
    from audiocraft_b200.encodec import CompressionModel, HFEncodecCompressionModel
    if rate == 48:
        hf = GO.hf_48k_model(seed=3)
    else:
        torch.manual_seed(3)
        hf = HFModel(EncodecConfig()).eval()
    hf.save_pretrained(str(tmp_path))
    m = CompressionModel.get_pretrained(str(tmp_path))
    assert isinstance(m, HFEncodecCompressionModel)
    assert (m.sample_rate, m.channels, m.frame_rate) == (rate * 1000, 2 if rate == 48 else 1, rate * 1000 / 320)
    x = H.audio_input(dict(sample_rate=rate * 1000, channels=m.channels), 1, 9000, 2)
    with torch.no_grad():
        ref = hf.encode(x, None, hf.config.target_bandwidths[-1], return_dict=False)[0][0]
    codes, _ = m.encode(x)
    assert (codes.cpu() == ref).float().mean() > 0.99
    with pytest.raises(FileNotFoundError):
        CompressionModel.get_pretrained('facebook/encodec_48khz')
