"""CPU tests of the MusicGen-melody host front-end: the chroma filter bank (held to properties: librosa is not a dependency),
the chroma extractor, ChromaStemConditioner, wav collation, the prepend fuser and the loader's chroma2music support."""
import math

import pytest
import torch

from audiocraft_b200 import conditioners as CD
from audiocraft_b200 import loaders, synth

SR, NFFT = 32000, 2 ** 14


def _tone(f, seconds=1.0, sr=SR):
    t = torch.arange(int(sr * seconds)) / sr
    return (0.3 * torch.sin(2 * math.pi * f * t))[None, None]


def test_filter_bank_shape_and_norms():
    fb = CD.chroma_filter_bank(SR, NFFT)
    assert fb.shape == (12, NFFT // 2 + 1) and fb.dtype == torch.float32
    assert bool((fb >= 0).all())


@pytest.mark.parametrize('f', [110.0, 196.0, 261.63, 440.0, 466.16, 659.25, 987.77, 1661.2])
def test_filter_bank_pure_tone_pitch_class(f):
    """base_c: row 0 is C, so A4 = 440 Hz is class 9 and f is class round(12 log2(f / 440)) + 9 mod 12."""
    fb = CD.chroma_filter_bank(SR, NFFT)
    col = int(round(f * NFFT / SR))
    assert int(fb[:, col].argmax()) == (round(12 * math.log2(f / 440.0)) + 9) % 12


def test_filter_bank_octave_weighting_centred_on_octave_5():
    """Each column's weight follows exp(-0.5 ((octs - 5) / 2)^2): largest near octave 5 (A440 / 16 * 2^5 = 880 Hz) and
    symmetric in octaves around it, and a tone one octave away maps to the same class."""
    fb = CD.chroma_filter_bank(SR, NFFT)

    def peak(f):
        return float(fb[:, int(round(f * NFFT / SR))].max())
    assert peak(880.0) > peak(440.0) and peak(880.0) > peak(1760.0)
    assert abs(peak(440.0) - peak(1760.0)) / peak(880.0) < 0.05
    for f in (220.0, 293.66, 392.0):
        c1 = int(fb[:, int(round(f * NFFT / SR))].argmax())
        c2 = int(fb[:, int(round(2 * f * NFFT / SR))].argmax())
        assert c1 == c2


def test_chroma_extractor_matches_torchaudio_spectrogram_and_frames():
    torchaudio = pytest.importorskip('torchaudio')
    ce = CD.ChromaExtractor(SR, 12, 14, argmax=True)
    wav = torch.randn(2, 1, SR)
    ref = torchaudio.transforms.Spectrogram(n_fft=NFFT, win_length=NFFT, hop_length=NFFT // 4, power=2, center=True,
                                            pad=0, normalized=True)(wav)
    torch.testing.assert_close(ce.spectrogram(wav), ref, rtol=1e-5, atol=1e-6)
    assert ce(torch.zeros(1, 1, 30 * SR)).shape == (1, 1 + 960000 // 4096, 12)
    out = ce(_tone(440.0, 2.0))
    assert bool((out.sum(-1) == 1).all()) and bool((out.argmax(-1) == 9).all())
    assert ce(torch.zeros(1, 1, 1)).shape == (1, 5, 12)   # a nullified wav is padded to one FFT window


def _conditioner(match_len, dim=16):
    c = CD.ChromaStemConditioner(dim, SR, 12, 14, 2.0, match_len_on_eval=match_len,
                                 stem_separator=CD.identity_stem_separator)
    torch.nn.init.normal_(c.output_proj.weight)
    return c


def _wav_attr(wav):
    return CD.ConditioningAttributes(text={}, wav={'self_wav': CD.WavCondition(
        wav, torch.tensor([wav.shape[-1]]), [SR], [None])})


def test_chroma_stem_conditioner_repeat_truncate_and_masking():
    c = _conditioner(True)
    assert c.chroma_len == 1 + 2 * SR // 4096
    prov = CD.ConditioningProvider({'self_wav': c})
    short, long = _tone(261.63, 0.5), _tone(261.63, 3.0)
    tok = prov.tokenize([_wav_attr(short)])
    emb, mask = prov(tok)['self_wav']
    assert emb.shape == (1, c.chroma_len, 16) and bool((mask == 1).all())
    chroma = c._get_wav_embedding(tok['self_wav'])
    n = c.chroma(short).shape[1]   # frames of the short wav itself (padded to one FFT window)
    torch.testing.assert_close(chroma[:, n:2 * n], chroma[:, :n])   # repeated periodically
    assert c._get_wav_embedding(prov.tokenize([_wav_attr(long)])['self_wav']).shape[1] == c.chroma_len   # truncated
    # masking (match_len_on_eval=False): a short wav padded in the batch is masked past its length / hop
    c2 = _conditioner(False)
    prov2 = CD.ConditioningProvider({'self_wav': c2})
    emb, mask = prov2(prov2.tokenize([_wav_attr(short), _wav_attr(long)]))['self_wav']
    lens = torch.tensor([short.shape[-1], long.shape[-1]]) / 4096
    assert torch.equal(mask.bool(), torch.arange(emb.shape[1])[None] < lens[:, None])
    assert bool((emb[0, int(lens[0]) + 1:] == 0).all())


def test_null_wav_conditions():
    c = _conditioner(False)
    prov = CD.ConditioningProvider({'self_wav': c})
    nulls = CD.nullify_all([_wav_attr(_tone(440.0, 0.5))])
    tok = prov.tokenize(nulls)
    assert tok['self_wav'].wav.shape == (1, 1, 1)
    emb, mask = prov(tok)['self_wav']
    assert bool((emb == 0).all()) and bool((mask == 0).all())


def test_collate_pads_to_longest_and_mixes_to_mono():
    prov = CD.ConditioningProvider({'self_wav': _conditioner(False)})
    a = torch.randn(1, 2, 100)
    b = torch.randn(1, 1, 40)
    out = prov._collate_wavs([_wav_attr(a), _wav_attr(b)])['self_wav']
    assert out.wav.shape == (2, 1, 100) and out.length.tolist() == [100, 40] and out.sample_rate == [SR, SR]
    torch.testing.assert_close(out.wav[0, 0], a.mean(1)[0])
    assert bool((out.wav[1, 0, 40:] == 0).all())


def test_fuser_prefix_order_chroma_then_description():
    fz = CD.ConditionFuser({'prepend': ['self_wav', 'description'], 'cross': []})
    desc = (torch.full((2, 3, 4), 1.0), torch.ones(2, 3))
    wav = (torch.full((2, 5, 4), 2.0), torch.ones(2, 5))
    out = fz.prefix_source({'description': desc, 'self_wav': wav})   # provider order: text, then wav
    assert out.shape == (2, 8, 4)
    assert bool((out[:, :5] == 2).all()) and bool((out[:, 5:] == 1).all())
    assert fz.cross_source({'description': desc, 'self_wav': wav}) is None
    assert CD.ConditionFuser({'prepend': ['self_wav']}).prefix_source({'self_wav': wav}).shape == (2, 5, 4)
    for bad in ({'sum': ['description']}, {'input_interpolate': ['self_wav']}):
        with pytest.raises(NotImplementedError):
            CD.ConditionFuser(bad)


def _xp(**over):
    xp = {
        'sample_rate': 32000,
        'dataset': {'segment_duration': 30},
        'transformer_lm': dict(dim=64, num_heads=1, num_layers=1, n_q=4, card=32, norm_first=True),
        'codebooks_pattern': {'modeling': 'delay', 'delay': {'delays': [0, 1, 2, 3]}},
        'classifier_free_guidance': {'inference_coef': 3.0},
        'fuser': {'cross_attention_pos_emb': False, 'sum': [], 'prepend': ['self_wav', 'description'], 'cross': [],
                  'input_interpolate': []},
        'conditioners': {
            'self_wav': {'model': 'chroma_stem', 'chroma_stem': dict(sample_rate=32000, n_chroma=12, radix2_exp=14,
                                                                     argmax=True, match_len_on_eval=False, eval_wavs=None,
                                                                     n_eval_wavs=100, cache_path=None)},
            'description': {'model': 't5', 't5': {'name': 't5-base'}}},
    }
    for k, v in over.items():
        sect, key = k.split('.', 1) if '.' in k else (k, None)
        if key is None:
            xp[sect] = v
        elif sect == 'chroma':
            xp['conditioners']['self_wav']['chroma_stem'][key] = v
        else:
            xp[sect][key] = v
    return xp


def test_loader_accepts_chroma2music():
    cfg = loaders.lm_cfg_from_xp(_xp())
    assert cfg['cross_attention'] is False and cfg['prepend'] == ['self_wav', 'description'] and cfg['cond_dim'] == 768
    assert cfg['chroma'] == dict(n_chroma=12, radix2_exp=14, argmax=True, match_len_on_eval=False, sample_rate=32000,
                                 duration=30.0)
    assert loaders.lm_cfg_from_xp(_xp(**{'fuser.prepend': ['self_wav']}))['prepend'] == ['self_wav']


@pytest.mark.parametrize('over', [{'fuser.sum': ['description']}, {'fuser.input_interpolate': ['self_wav']},
                                  {'fuser.prepend': ['description']}, {'chroma.eval_wavs': 'egs/eval.jsonl'},
                                  {'chroma.cache_path': '/tmp/cache'}])
def test_loader_refusals(over):
    with pytest.raises(NotImplementedError):
        loaders.lm_cfg_from_xp(_xp(**over))


def test_loader_needs_a_stem_separator(tmp_path):
    import yaml
    cfg = synth.lm_config('lm_mini_melody')
    xp = _xp(transformer_lm=dict(dim=cfg['dim'], num_heads=cfg['num_heads'], num_layers=cfg['num_layers'], n_q=4,
                                 card=cfg['card'], norm_first=True))
    path = tmp_path / 'state_dict.bin'
    torch.save({'best_state': {}, 'xp.cfg': yaml.safe_dump(xp)}, str(path))
    with pytest.raises(RuntimeError, match='stem_separator'):
        loaders.load_lm_model(str(path), device='cpu', text_encoder=lambda e: None)
    with pytest.raises(RuntimeError, match='stem_separator'):
        CD.ChromaStemConditioner(16, SR, 12, 14, 1.0)


def test_synthetic_melody_config():
    cfg = synth.lm_config('musicgen_melody')
    assert (cfg['dim'], cfg['num_heads'], cfg['num_layers'], cfg['cross_attention'], cfg['cond_dim'], cfg['n_chroma'],
            cfg['radix2_exp']) == (1536, 24, 48, False, 768, 12, 14)
    sd = synth.synth_lm_state_dict(synth.lm_config('lm_mini_melody'), seed=0)
    assert sd['condition_provider.conditioners.self_wav.output_proj.weight'].shape == (256, 12)
    assert not any('cross_attention' in k for k in sd)


# ----------------------------------------------------------------------------- against the reference's melody modules
from tests import melody_golden as MG  # noqa: E402
from tests.prefix_oracle import PrefixLMOracle  # noqa: E402

_G = MG.golden()


@pytest.mark.parametrize('case', list(_G['cases']))
def test_conditioners_match_reference_golden(case):
    """Chroma (one-hot per frame, masking / repeat / truncate / null wavs) exactly, the [chroma ; description] prefix after
    output_proj within 5e-5, as the reference's ChromaStemConditioner, T5 stand-in and prepend fuser produce them."""
    c = _G['cases'][case]
    cfg = MG.config(_G, case)
    sd = MG.weights(_G, cfg)
    chroma, mask, prefix = MG.repo_conditions(_G, case, cfg, sd)
    assert torch.equal(chroma, c['chroma'])
    assert torch.equal(mask.long(), c['self_wav_mask'].long())
    assert prefix.shape[1] == c['prefix_len']
    torch.testing.assert_close(prefix[..., ::c['prefix_stride']], c['prefix_strided'], rtol=0, atol=5e-5)


@pytest.mark.parametrize('case', list(_G['cases']))
def test_prefix_oracle_matches_reference_golden(case):
    """The fp32 prefix oracle on this package's prefix: teacher-forced CFG logits within 5e-5 of the reference's
    LMModel.forward with the prepend fuser, greedy tokens equal to its generate()."""
    c = _G['cases'][case]
    cfg = MG.config(_G, case)
    sd = MG.weights(_G, cfg)
    _, _, prefix = MG.repo_conditions(_G, case, cfg, sd)
    o = PrefixLMOracle(sd, cfg, half_gemm=False, prefix=prefix)
    lg = o.teacher_forced_mixed(MG.teacher_sequence(_G, cfg), None, cfg['cfg_coef'])
    torch.testing.assert_close(lg[..., c['logits_idx']], c['logits'], rtol=0, atol=5e-5)
    out = o.generate(None, None, _G['batch'], _G['T'], use_sampling=False)
    assert torch.equal(out, c['greedy'])
