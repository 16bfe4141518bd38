"""Pin the CPU oracle (oracle/) to outputs of the REAL reference modules (tests/golden/*.pt, produced by
tests/golden/make_golden.py on the CPU).  Integer outputs must match exactly; float outputs to
fp32 round-off (tolerances written at each check)."""
import os

import pytest
import torch

from tests import helpers as H
from audiocraft_b200 import synth
from oracle import encodec_oracle as EO, lm_oracle as LO


def _load(name):
    return torch.load(os.path.join(H.GOLDEN_DIR, name), weights_only=False)


@pytest.mark.parametrize('name', ['encodec_tiny', 'encodec_tiny_causal', 'encodec_24k', 'encodec_32k'])
def test_encodec_oracle_matches_reference(name):
    g = _load(f'{name}.pt')
    cfg = synth.ENCODEC_CONFIGS[name]
    sd = synth.synth_encodec_state_dict(cfg, seed=g['wseed'])
    x = H.audio_input(cfg, g['batch'], g['length'], g['xseed'])
    assert torch.equal(x[..., :64], g['x_head']), "seeded input is not reproducible on this torch build"
    o = EO.EncodecOracle(sd, cfg)
    codes, scale = o.encode(x)
    assert codes.dtype == torch.int64
    assert torch.equal(codes, g['codes'])  # bit-exact RVQ indices
    if g['scale'] is None:
        assert scale is None
    else:
        torch.testing.assert_close(scale, g['scale'], rtol=1e-6, atol=0)
    lat = o.encode_latent(o.preprocess(x)[0])
    torch.testing.assert_close(lat, g['latent'], rtol=0, atol=2e-5)
    wav = o.decode(g['codes'], g['scale'])
    if 'wav' in g:
        torch.testing.assert_close(wav, g['wav'], rtol=0, atol=2e-5)
        torch.testing.assert_close(o.decode_latent(g['codes']), g['qlat'], rtol=0, atol=1e-6)
    else:
        assert wav.shape[-1] == g['wav_len']
        torch.testing.assert_close(wav[..., :512], g['wav_head'], rtol=0, atol=2e-5)
        torch.testing.assert_close(wav[..., ::g['wav_stride']], g['wav_strided'], rtol=0, atol=2e-5)


def _lm_setup(name, g):
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=g['wseed'])
    _, _, cross = H.lm_condition(cfg, sd, g['batch'], g['t_text'], g['cseed'])
    return cfg, sd, cross


@pytest.mark.parametrize('name', ['lm_mini', 'lm_tiny'])
def test_lm_oracle_matches_reference(name):
    g = _load(f'{name}.pt')
    cfg, sd, cross = _lm_setup(name, g)
    o = LO.LMOracle(sd, cfg)
    B, T = g['batch'], g['T']
    logits = []
    out = o.generate(None, cross, B, T, use_sampling=False, record_logits=logits)
    assert torch.equal(out, g['greedy'])
    n = g['logits'].shape[0]
    torch.testing.assert_close(torch.stack(logits[:n]), g['logits'], rtol=0, atol=5e-5)
    # torch-generator sampling reproduces the reference's torch.multinomial stream (utils/utils.py:103)
    for key, seed, kw in [('sampled_topk', 11, dict(top_k=10, temp=0.9)),
                          ('sampled_topp', 12, dict(top_k=0, top_p=0.8)),
                          ('sampled_plain', 13, dict(top_k=0, top_p=0.0, temp=1.3))]:
        gen = torch.Generator()
        gen.manual_seed(seed)
        got = o.generate(None, cross, B, T, use_sampling=True, generator=gen, **kw)
        assert torch.equal(got, g[key]), key
    got = o.generate(g['greedy'][..., :5].clone(), cross, B, T, use_sampling=False)
    assert torch.equal(got, g['continuation'])
    got = o.generate(None, torch.zeros_like(cross), B, T, use_sampling=False)
    assert torch.equal(got, g['unconditional'])


@pytest.mark.slow
def test_lm_oracle_matches_reference_musicgen_small():
    g = _load('musicgen_small.pt')
    cfg, sd, cross = _lm_setup('musicgen_small', g)
    o = LO.LMOracle(sd, cfg)
    logits = []
    out = o.generate(None, cross, g['batch'], g['T'], use_sampling=False, record_logits=logits)
    assert torch.equal(out, g['greedy'])
    lg = torch.stack(logits[:g['logits_top_v'].shape[0]])
    torch.testing.assert_close(lg.gather(-1, g['logits_top_i']), g['logits_top_v'], rtol=0, atol=2e-4)


def test_patterns_match_reference():
    g = _load('patterns.pt')
    for (K, T, delays), ref in g.items():
        seq, mask = LO.build_delay_sequence(ref['codes'], list(delays), 99)
        assert torch.equal(seq, ref['seq']) and torch.equal(mask, ref['mask'])
        back, bmask = LO.revert_delay_sequence(seq, list(delays), -1, T)
        assert torch.equal(back, ref['back']) and torch.equal(bmask, ref['back_mask'])
        assert torch.equal(back, ref['codes'])  # round trip
        assert ref['first_step_T0'] == [t + 1 + min(delays) for t in range(T)]


def test_sampling_matches_reference():
    g = _load('sampling.pt')
    gen = torch.Generator()
    gen.manual_seed(g['seed'])
    probs = torch.softmax(torch.randn(6, 4, 2048, generator=gen) * 2.0, -1)
    torch.manual_seed(31)
    assert torch.equal(LO.multinomial(LO.top_k_filter(probs.clone(), 250)), g['top_k_250'])
    torch.manual_seed(32)
    ps, pi = LO.top_p_sorted(probs.clone(), 0.9)
    assert torch.equal(torch.gather(pi, -1, LO.multinomial(ps)), g['top_p_0.9'])
    torch.manual_seed(33)
    assert torch.equal(LO.multinomial(probs.clone()), g['plain'])
    # injected-noise formulation == torch.multinomial for an identically seeded generator
    g1, g2 = torch.Generator(), torch.Generator()
    g1.manual_seed(5)
    g2.manual_seed(5)
    flat = probs.reshape(-1, 2048)
    noise = torch.empty_like(flat).exponential_(1, generator=g1)
    assert torch.equal(LO.multinomial_with_noise(probs, noise), LO.multinomial(probs, generator=g2))


def test_padding_rules():
    """Shape algebra pinned by the reference's own tests (tests/modules/test_conv.py:160-203,
    tests/modules/test_seanet.py:18-56): conv output length ceil(L/s), convtr length L*s after trimming."""
    import math
    for (k, s, d) in [(4, 1, 1), (4, 2, 1), (3, 1, 3), (10, 5, 1), (3, 2, 3)]:
        for causal in (False, True):
            for L in (1, 2, 7, 50, 51, 333):
                x = torch.randn(1, 2, L)
                y = EO.sconv1d(x, torch.randn(3, 2, k), torch.zeros(3), stride=s, dilation=d, causal=causal)
                assert y.shape[-1] == math.ceil(L / s), (k, s, d, causal, L)
    for (k, s) in [(8, 4), (10, 5), (16, 8), (4, 2)]:
        for causal, ratio in [(False, 1.0), (True, 1.0), (True, 0.5), (True, 0.0)]:
            y = EO.sconvtr1d(torch.randn(1, 2, 13), torch.randn(2, 3, k), torch.zeros(3), s, causal, ratio)
            assert y.shape[-1] == 13 * s


@pytest.mark.parametrize('shortcut', [False, True])
def test_oracle_matches_huggingface_encodec(shortcut):
    """Third-party arithmetic at the boundary (SURVEY section 8c): `facebook/encodec_*` goes through
    transformers.EncodecModel (audiocraft/models/encodec.py:119-121).  transformers is in the image, so HF's own CPU
    implementation (random init; no checkpoints offline) pins the oracle a second time, through the key conversion."""
    import warnings
    from transformers import EncodecConfig, EncodecModel
    from audiocraft_b200.encodec import hf_encodec_to_reference
    warnings.filterwarnings('ignore')
    hc = EncodecConfig(use_conv_shortcut=shortcut)
    torch.manual_seed(0)
    m = EncodecModel(hc).eval()
    hsd = m.state_dict()
    g = torch.Generator().manual_seed(1)
    for k in hsd:
        if k.endswith('codebook.embed'):
            hsd[k].copy_(torch.randn(hsd[k].shape, generator=g) * 0.5)
    sd, cfg = hf_encodec_to_reference(hsd, hc)
    assert cfg['possible_num_codebooks'] == [2, 4, 8, 16, 32] and cfg['true_skip'] == (not shortcut)
    x = torch.randn(2, 1, 3000, generator=g) * 0.3
    with torch.no_grad():
        enc = m.encode(x, None, 24.0)
        dec = m.decode(enc[0], enc[1])[0]
    o = EO.EncodecOracle(sd, cfg)
    codes, scale = o.encode(x)
    assert scale is None and torch.equal(codes, enc[0][0])
    torch.testing.assert_close(o.decode(codes), dec, rtol=0, atol=2e-6)


@pytest.mark.parametrize('pe', ['rope', 'sin_rope'])
def test_lm_oracle_rope_matches_reference(pe):
    """Rotary positions (rope.py:84-125): teacher-forced logits of one causal forward and streaming greedy tokens."""
    g = _load('lm_mini_rope.pt')
    cfg = synth.lm_config('lm_mini')
    cfg['positional_embedding'], cfg['positional_scale'] = pe, g['positional_scale']
    sd = synth.synth_lm_state_dict(cfg, seed=g['wseed'])
    B, T = g['batch'], g['T']
    _, _, cross = H.lm_condition(cfg, sd, B, g['t_text'], g['cseed'])
    seq = H.fullsize_sequence(cfg, B, T, g['sseed'])
    o = LO.LMOracle(sd, cfg)
    o.reset()
    outs = [o.forward(torch.cat([seq, seq], 0)[..., t:t + 1], cross) for t in range(seq.shape[-1] - 1)]   # streaming
    lg = torch.cat(outs, dim=2)
    c, u = lg.split(B, dim=0)
    mixed = (u + (c - u) * cfg['cfg_coef']).permute(2, 0, 1, 3)
    torch.testing.assert_close(mixed, g[pe]['logits'], rtol=0, atol=5e-5)
    assert torch.equal(o.generate(None, cross, B, T, use_sampling=False), g[pe]['greedy'])


@pytest.mark.slow
@pytest.mark.parametrize('name', ['musicgen_medium', 'musicgen_large'])
def test_lm_oracle_fulldepth_matches_reference(name):
    """Full-depth released architectures over 1500 frames (tests/golden/*_full.pt): minutes of CPU per model, so only
    with ACB_SLOW_TESTS=1 (the GPU suite checks the CUDA path against the same fixtures, tests/test_gpu_fullsize.py)."""
    import os as _os
    if _os.environ.get('ACB_SLOW_TESTS') != '1':
        pytest.skip('set ACB_SLOW_TESTS=1 (about 10 CPU-minutes per model)')
    g = _load(f'{name}_full.pt')
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=g['wseed'])
    B = g['batch']
    _, _, cross = H.lm_condition(cfg, sd, B, g['t_text'], g['cseed'])
    seq = H.fullsize_sequence(cfg, B, g['T'], g['sseed'])
    o = LO.LMOracle(sd, cfg)
    lg = o.forward(torch.cat([seq, seq], 0)[..., :-1], cross)
    c, u = lg.split(B, dim=0)
    mixed = (u + (c - u) * cfg['cfg_coef'])[:, :, g['steps'], :].permute(2, 0, 1, 3)
    torch.testing.assert_close(mixed.gather(-1, g['logits_top_i'].long()), g['logits_top_v'], rtol=0, atol=2e-4)
