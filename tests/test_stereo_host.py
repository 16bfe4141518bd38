"""CPU tests of stereo MusicGen: the stereo checkpoints' xp.cfg, the synthetic stereo architectures, and the CPU oracles against
the reference's own stereo modules (tests/golden/lm_mini_stereo.pt, written by tests/golden/make_golden_stereo.py).

Integer outputs must match exactly, float outputs to fp32 round-off (5e-5 for the LM, 2e-5 for the codec, as in
tests/test_oracle_vs_golden.py)."""
import os

import pytest
import torch
import yaml

from tests import helpers as H
from audiocraft_b200 import loaders, synth
from audiocraft_b200.patterns import DelayedPatternProvider
from oracle import encodec_oracle as EO, lm_oracle as LO

STEREO_DELAYS = [0, 0, 1, 1, 2, 2, 3, 3]


def _golden():
    return torch.load(os.path.join(H.GOLDEN_DIR, 'lm_mini_stereo.pt'), weights_only=False)


def _stereo_xp(melody=False, **isc):
    """The fields of a released musicgen-stereo-* xp.cfg that the loaders read (config/solver/musicgen/default.yaml:20-29,
    docs/MUSICGEN.md "Training stereo models")."""
    xp = {
        'sample_rate': 32000, 'channels': 2,
        'dataset': {'segment_duration': 30},
        'transformer_lm': dict(dim=1024, num_heads=16, num_layers=24, n_q=8, card=2048, norm_first=True),
        'codebooks_pattern': {'modeling': 'delay', 'delay': {'delays': list(STEREO_DELAYS)}},
        'classifier_free_guidance': {'inference_coef': 3.0},
        'interleave_stereo_codebooks': dict({'use': True, 'per_timestep': False}, **isc),
        'compression_model_n_q': 4,
        'fuser': {'cross_attention_pos_emb': False, 'sum': [], 'prepend': [], 'cross': ['description'],
                  'input_interpolate': []},
        'conditioners': {'description': {'model': 't5', 't5': {'name': 't5-base'}}},
    }
    if melody:
        xp['fuser'].update(prepend=['self_wav', 'description'], cross=[])
        xp['conditioners']['self_wav'] = {'model': 'chroma_stem', 'chroma_stem': dict(
            sample_rate=32000, n_chroma=12, radix2_exp=14, argmax=True, match_len_on_eval=True, eval_wavs=None, cache_path=None)}
    return xp


class _MonoCodec:
    """The CompressionModel surface InterleaveStereoCompressionModel reads, without a device: encodec_32k's properties."""
    channels, cardinality, frame_rate, sample_rate, total_codebooks = 1, 2048, 50, 32000, 4

    def __init__(self):
        self.num_codebooks = 4

    def set_num_codebooks(self, n):
        assert 0 < n <= self.total_codebooks
        self.num_codebooks = n


@pytest.mark.parametrize('melody', [False, True])
def test_stereo_xp_cfg_parses(tmp_path, melody):
    xp = _stereo_xp(melody)
    cfg = loaders.lm_cfg_from_xp(xp)
    assert cfg['n_q'] == 8 and cfg['card'] == 2048 and cfg['delays'] == STEREO_DELAYS
    assert cfg['cross_attention'] is not melody and cfg['prepend'] == (['self_wav', 'description'] if melody else [])
    path = tmp_path / 'state_dict.bin'
    torch.save({'best_state': {}, 'xp.cfg': yaml.safe_dump(xp)}, str(path))
    cm = loaders._wrap_from_xp(_MonoCodec(), str(path))
    assert (cm.channels, cm.num_codebooks, cm.cardinality, cm.frame_rate, cm.sample_rate) == (2, 8, 2048, 50, 32000)
    assert cm.num_codebooks == cfg['n_q']


def test_per_timestep_interleaving_is_refused():
    with pytest.raises(NotImplementedError, match='per_timestep'):
        loaders.lm_cfg_from_xp(_stereo_xp(per_timestep=True))
    # `use: false` is a mono checkpoint whatever per_timestep says
    assert loaders.lm_cfg_from_xp(_stereo_xp(use=False, per_timestep=True))['n_q'] == 8


@pytest.mark.parametrize('scale,mono', [('stereo-small', 'musicgen_small'), ('stereo-medium', 'musicgen_medium'),
                                        ('stereo-large', 'musicgen_large'), ('stereo-melody', 'musicgen_melody'),
                                        ('stereo-melody-large', None)])
def test_synthetic_stereo_architectures(scale, mono):
    """`synthetic/stereo-<scale>` names the mono widths at 8 codebooks on the paired delays; the melody ones keep the chroma
    prefix and no cross attention (musicgen-stereo-melody-large has MusicGen-large's width)."""
    cfg = synth.lm_config(loaders._SCALES[scale])
    ref = synth.lm_config(mono) if mono else dict(synth.lm_config('musicgen_large'), **{
        k: synth.lm_config('musicgen_melody')[k] for k in ('cross_attention', 'cond_dim', 'n_chroma', 'radix2_exp')})
    assert cfg['n_q'] == 8 and cfg['delays'] == STEREO_DELAYS and cfg['card'] == 2048
    for k in ('dim', 'num_heads', 'num_layers', 'hidden_scale', 'cross_attention', 'cond_dim', 'n_chroma'):
        assert cfg.get(k) == ref.get(k), k


@pytest.mark.parametrize('name', ['lm_mini_stereo', 'lm_mini_melody_stereo'])
def test_stereo_state_dict_layout(name):
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=0)
    d, card = cfg['dim'], cfg['card']
    assert sorted(k for k in sd if k.startswith('emb.')) == [f'emb.{k}.weight' for k in range(8)]
    assert sorted(k for k in sd if k.startswith('linears.')) == [f'linears.{k}.weight' for k in range(8)]
    assert all(sd[f'emb.{k}.weight'].shape == (card + 1, d) and sd[f'linears.{k}.weight'].shape == (card, d) for k in range(8))
    assert ('condition_provider.conditioners.self_wav.output_proj.weight' in sd) == bool(cfg.get('n_chroma'))


def _mini():
    g = _golden()
    cfg = synth.lm_config(g['name'])
    sd = synth.synth_lm_state_dict(cfg, seed=g['wseed'])
    _, _, cross = H.lm_condition(cfg, sd, g['batch'], g['t_text'], g['cseed'])
    return g, cfg, sd, cross


def test_oracle_reproduces_lm_mini_stereo_golden():
    """Greedy tokens and a greedy continuation exactly; the CFG-mixed teacher-forced logits within 5e-5."""
    g, cfg, sd, cross = _mini()
    B, T = g['batch'], g['T']
    o = LO.LMOracle(sd, cfg)
    assert torch.equal(o.generate(None, cross, B, T, use_sampling=False), g['greedy'])
    assert torch.equal(o.last_sequence, g['sequence'])
    P = g['prompt_len']
    assert torch.equal(o.generate(g['greedy'][..., :P].clone(), cross, B, T, use_sampling=False), g['continuation'])
    seq = g['sequence']
    o.reset()
    c, u = o.forward(torch.cat([seq, seq], 0)[..., :-1], cross).split(B, dim=0)
    mixed = (u + (c - u) * cfg['cfg_coef']).permute(2, 0, 1, 3)
    torch.testing.assert_close(mixed[..., g['logits_idx']], g['logits'], rtol=0, atol=5e-5)
    assert torch.equal(mixed.argmax(-1), g['logits_argmax'].long())


def test_oracle_compute_predictions_match_lm_mini_stereo_golden():
    """LMModel.compute_predictions on stereo codes: the pattern's [B, 8, T, card] logits, NaN pattern and mask."""
    g, cfg, sd, cross = _mini()
    p, B = g['predictions'], g['batch']
    codes = torch.randint(0, cfg['card'], (B, 8, p['T']), generator=torch.Generator().manual_seed(p['kseed']))
    pattern = DelayedPatternProvider(8, delays=cfg['delays']).get_pattern(p['T'])
    o = LO.LMOracle(sd, cfg)
    for key, valid in (('valid', True), ('all', False)):
        seq = pattern.build_pattern_sequence(codes, cfg['card'], keep_only_valid_steps=valid)[0]
        o.reset()
        lg = o.forward(seq, cross[:B])                                                  # [B, 8, S, card]
        S = lg.shape[2]
        idx, mask = pattern.logits_tables(S, valid)
        flat = torch.cat([lg.reshape(B, 8 * S, -1), torch.full((B, 1, lg.shape[-1]), float('nan'))], dim=1)
        out = flat[:, torch.from_numpy(idx).reshape(-1)].reshape(B, 8, p['T'], -1)
        assert torch.equal(torch.from_numpy(mask), p[f'mask_{key}'])
        assert torch.equal(torch.isnan(out).all(-1), p[f'nan_{key}']) and torch.equal(torch.isnan(out).any(-1), p[f'nan_{key}'])
        torch.testing.assert_close(out[..., g['logits_idx']], p[f'logits_{key}'], rtol=0, atol=5e-5, equal_nan=True)
        ok = ~p[f'nan_{key}']
        torch.testing.assert_close(out.gather(-1, p[f'top_i_{key}'].long())[ok], p[f'top_v_{key}'][ok], rtol=0, atol=5e-5)


def test_oracle_stereo_codec_matches_golden():
    """The reference's InterleaveStereoCompressionModel over encodec_32k: both channels through the mono oracle, codes
    interleaved `b (k c) t`, and the decode of the golden codes."""
    c = _golden()['codec']
    cfg = synth.ENCODEC_CONFIGS[c['name']]
    o = EO.EncodecOracle(synth.synth_encodec_state_dict(cfg, seed=c['wseed']), cfg)
    x = H.audio_input(dict(cfg, channels=2), c['codes'].shape[0], c['length'], c['xseed'])
    assert torch.equal(x[..., :64], c['x_head'])
    B = x.shape[0]
    codes, scale = o.encode(x.transpose(0, 1).reshape(2 * B, 1, -1))
    assert scale is None
    inter = codes.view(2, B, 4, -1).permute(1, 2, 0, 3).reshape(B, 8, -1)
    assert torch.equal(inter, c['codes'])
    assert c['props'] == (8, 50, 2, 2048, 4)
    left, right = c['codes'].view(B, 4, 2, -1).unbind(2)
    wav = torch.cat([o.decode(left), o.decode(right)], dim=1)
    assert wav.shape == (B, 2, c['wav_len'])
    torch.testing.assert_close(wav[..., ::c['wav_stride']], c['wav_strided'], rtol=0, atol=2e-5)
