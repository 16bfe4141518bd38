"""EnCodec 48 kHz and GroupNorm codecs, host side (no GPU): the transformers -> reference conversion, the refusal of norms the
kernels do not run, the chunk geometry, and the CPU oracle against transformers' model and the reference's own GroupNorm
EnCodec (tests/golden/encodec_tiny_gn.pt)."""
import os

import pytest
import torch

from audiocraft_b200 import synth
from audiocraft_b200.encodec import EncodecModel, check_norm, chunk_bounds, hf_encodec_to_reference
from oracle import encodec_oracle as EO
from tests import encodec_gn_oracle as GO
from tests import helpers as H

pytest.importorskip('transformers')


def test_hf_48k_conversion_matches_reference_layout():
    """Every converted key is a key of the reference's GroupNorm EncodecModel of the same architecture, with its shape."""
    hf = GO.hf_48k_model()
    sd, cfg = hf_encodec_to_reference(hf.state_dict(), hf.config)
    want = synth.synth_encodec_state_dict(synth.ENCODEC_GN_CONFIGS['encodec_48k'], 0)
    assert set(sd) == set(want)
    assert all(sd[k].shape == want[k].shape for k in sd)
    assert sum(k.endswith('.norm.weight') for k in sd) == 2 * 1 + 4 * 4 + 2 + 4 * 4   # first/last convs, 4 stages x (3 convs + shortcut)
    ref = dict(synth.ENCODEC_GN_CONFIGS['encodec_48k'])
    for k in ('channels', 'n_filters', 'ratios', 'causal', 'pad_mode', 'lstm', 'norm', 'true_skip', 'sample_rate', 'n_q', 'bins',
              'renormalize'):
        assert cfg[k] == ref[k], k
    assert (cfg['chunk_length'], cfg['chunk_stride'], cfg['possible_num_codebooks']) == (48000, 47520, [2, 4, 8, 16])
    assert cfg['norm_params'] == {'eps': 1e-5} and check_norm(cfg) == 1e-5
    # gamma is [C_out] of the conv it follows, for the transposed convs too
    assert sd['decoder.model.3.convtr.norm.weight'].shape == (256,)
    assert torch.equal(sd['decoder.model.3.convtr.norm.weight'], hf.state_dict()['decoder.layers.3.norm.weight'])


@pytest.mark.parametrize('over,exc', [
    (dict(norm='spectral_norm'), NotImplementedError),
    (dict(norm='layer_norm'), NotImplementedError),
    (dict(norm='time_group_norm', norm_params={'eps': 1e-5, 'affine': False}), NotImplementedError),
    (dict(norm='time_group_norm', causal=True), ValueError),
])
def test_unbuilt_norms_are_refused_before_the_device(over, exc):
    """These used to build a codec that ran without its norm; now they raise before any weight reaches a device."""
    cfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'], **over)
    with pytest.raises(exc):
        EncodecModel(synth.synth_encodec_state_dict(dict(cfg, norm='weight_norm'), 0), cfg, device='cpu')


def test_hf_unknown_norm_type_is_refused():
    hc = GO.hf_48k_config()
    hc.norm_type = 'layer_norm'
    with pytest.raises(NotImplementedError):
        hf_encodec_to_reference({}, hc)


def test_audiocraft_checkpoint_with_spectral_norm_is_refused(tmp_path):
    import yaml
    from audiocraft_b200.loaders import load_compression_model
    cfg = synth.ENCODEC_CONFIGS['encodec_tiny']
    xp = dict(channels=1, sample_rate=16000, encodec=dict(causal=False, renormalize=True),
              seanet=dict(dimension=32, n_filters=8, n_residual_layers=2, ratios=[5, 4, 2], kernel_size=7, last_kernel_size=7,
                          residual_kernel_size=3, dilation_base=2, pad_mode='reflect', compress=2, lstm=2, norm='spectral_norm',
                          norm_params={}),
              rvq=dict(n_q=4, bins=64))
    path = str(tmp_path / 'codec.bin')
    torch.save({'best_state': synth.synth_encodec_state_dict(dict(cfg, norm='none'), 0), 'xp.cfg': yaml.safe_dump(xp)}, path)
    with pytest.raises(NotImplementedError):
        load_compression_model(path, device='cpu')


@pytest.mark.parametrize('seconds', [0.5, 1.0, 3.0, 10.0])
def test_chunk_geometry_matches_transformers(seconds):
    hf = GO.hf_48k_model()
    L = int(seconds * 48000)
    x = torch.randn(1, 2, L) * 0.1
    b = chunk_bounds(L, hf.config.chunk_length, hf.config.chunk_stride)
    assert len(b) == -(-L // 47520)
    if seconds == 3.0:
        with torch.no_grad():
            codes, scales, pad = hf.encode(x, None, 3.0, return_dict=False)
        assert len(b) == 4 and codes.shape == (4, 1, 2, 150) and len(scales) == 4
        assert b[-1][1] - b[-1][0] == 1440 and -(-1440 // 320) == 5 and pad == 145


def test_gn_oracle_matches_transformers_48k():
    """The oracle's GroupNorm SEANet and chunk / overlap-add restatement against transformers' 48 kHz model: 3 s of stereo."""
    hf = GO.hf_48k_model()
    sd, cfg = hf_encodec_to_reference(hf.state_dict(), hf.config)
    x = H.audio_input(cfg, 1, 3 * 48000, 3)
    with torch.no_grad():
        codes, scales, pad = hf.encode(x, None, 24.0, return_dict=False)
        wav = hf.decode(codes, scales, None, False, pad)[0]
        lat = hf.encoder(x[..., :48000] / scales[0].view(-1, 1, 1))
    o_codes, o_scales, o_pad = GO.encode_chunks(x, sd, cfg, 16, 48000, 47520)
    assert o_pad == pad and torch.equal(o_codes, codes)
    for a, b in zip(o_scales, scales):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=0)
    torch.testing.assert_close(GO.encode_latent(x[..., :48000] / o_scales[0].view(-1, 1, 1), sd, cfg), lat, rtol=0, atol=5e-5)
    o_wav = GO.decode_chunks(o_codes, o_scales, sd, cfg, 47520, o_pad)
    assert o_wav.shape == wav.shape
    torch.testing.assert_close(o_wav, wav, rtol=0, atol=5e-5)


def test_gn_oracle_matches_reference_golden():
    g = torch.load(os.path.join(H.GOLDEN_DIR, 'encodec_tiny_gn.pt'), weights_only=False)
    cfg = g['cfg']
    sd = synth.synth_encodec_state_dict(cfg, seed=g['wseed'])
    x = H.audio_input(cfg, g['batch'], g['length'], g['xseed'])
    codes, scale, lat = GO.encode(x, sd, cfg, cfg['n_q'])
    torch.testing.assert_close(lat, g['latent'], rtol=0, atol=1e-5)
    torch.testing.assert_close(scale, g['scale'], rtol=1e-6, atol=0)
    _, margins = EO.rvq_encode(g['latent'], EO.codebooks_of(sd, cfg['n_q']), return_margin=True)
    neq = codes != g['codes']
    assert (margins[neq.int().cumsum(1).eq(1) & neq].abs() < 1e-4).all()
    wav = GO.decode(g['codes'], sd, cfg, g['scale'])
    assert wav.shape[-1] == g['wav_len']
    torch.testing.assert_close(wav[..., ::g['wav_stride']], g['wav_strided'], rtol=0, atol=1e-5)
