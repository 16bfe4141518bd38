"""T5 text encoder on the H100 (csrc/t5.cu, audiocraft_b200.t5, conditioners.T5Conditioner).

Against tests/golden/t5_conditioner.pt, the reference's own T5Conditioner in fp32 on CPU (tests/golden/make_golden_t5.py):
t5-base at full depth with ragged prompts, None / "" entries, the [cond; null] rows, a prompt past 128 tokens and hand-made
ids over the whole embedding; t5-large at full depth; and a "hot" t5-base whose ReLU activations pass fp16's range.  The
device GEMMs run on TF32 (10-bit mantissa operands, fp32 accumulation); a CPU emulation of that rounding on seeded t5-base
reached 3e-3 max / 5e-4 mean abs error on the hidden states, so the bounds are 1e-2 / 1e-3 there and 2e-2 on the outputs.
Then: null rows are exact zeros, a fully masked row passed straight to the C-ABI is zeros, an item is bit-identical alone
and in a padded batch, and MusicGen / AudioGen / a melody model generate from a local T5 directory exactly as from the
same conditioner's precomputed output.
"""
import os

import pytest
import torch

from audiocraft_b200 import synth
from tests import t5_golden as G

pytestmark = pytest.mark.gpu
os.environ.setdefault('HF_HUB_OFFLINE', '1')
pytest.importorskip('transformers')


@pytest.fixture(scope='module')
def golden():
    return torch.load(G.GOLDEN, weights_only=True)['cases']


@pytest.fixture(scope='module')
def t5_dirs(tmp_path_factory):
    """case -> a local HF-layout T5 directory holding that case's weights (t5-large as pytorch_model.bin)."""
    out = {}
    for name in G.CASES:
        cfg, sd = G.state_dict(name)
        path = str(tmp_path_factory.mktemp(f't5_{name}'))
        synth.write_t5_dir(path, cfg, sd, G.SPIECE, fmt='bin' if name == 'large' else 'safetensors')
        out[name] = path
    return out


def _conditioner(case, path):
    from audiocraft_b200.conditioners import T5Conditioner
    arch, _, _, out_dim, pseed = G.CASES[case][:5]
    cond = T5Conditioner(path, out_dim, device='cuda').to('cuda')
    pw, pb = G.proj_weights(synth.T5_CONFIGS[arch]['d_model'], out_dim, pseed)
    with torch.no_grad():
        cond.output_proj.weight.copy_(pw)
        cond.output_proj.bias.copy_(pb)
    return cond


def _check(what, got, want, idx, bound_max, bound_mean=None):
    got = got.reshape(got.shape[0], -1).gather(1, idx.to(got.device).long()).cpu()
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    err = (got - want).abs()
    print(f"{what}: max abs err {err.max():.3e}, mean {err.mean():.3e} (|ref| max {want.abs().max():.3g})")
    assert err.max() <= bound_max
    if bound_mean is not None:
        assert err.mean() <= bound_mean


@pytest.mark.parametrize('case', list(G.CASES))
def test_against_reference_conditioner(case, golden, t5_dirs):
    g = golden[case]
    cond = _conditioner(case, t5_dirs[case])
    descs = g['descs']
    inputs = cond.tokenize(descs + [None] * len(descs))
    assert torch.equal(inputs['input_ids'], g['ids']) and torch.equal(inputs['attention_mask'], g['mask'])
    emb, mask = cond(inputs)
    assert emb.is_cuda and emb.dtype == torch.float32 and torch.equal(mask.cpu(), g['mask'])
    live = g['mask'].any(1)
    assert bool((emb[~live.cuda()] == 0).all()), "null rows must be exact zeros"
    _check(f'{case} output', emb, g['emb'], g['emb_idx'], 2e-2)
    rows = live.nonzero().flatten()
    _, hid = cond.t5.encode(g['ids'][rows], g['mask'][rows], cond.output_proj.weight, cond.output_proj.bias, return_hidden=True)
    _check(f'{case} hidden', hid, g['hid'][rows], g['hid_idx'][rows], 1e-2, 1e-3)
    if 'hand' in g:   # ids spread over the whole embedding, ragged masks
        h = g['hand']
        emb, hid = cond.t5.encode(h['ids'], h['mask'], cond.output_proj.weight, cond.output_proj.bias, return_hidden=True)
        _check(f'{case} hand-made ids output', emb, h['emb'], h['emb_idx'], 2e-2)
        _check(f'{case} hand-made ids hidden', hid, h['hid'], h['hid_idx'], 1e-2, 1e-3)


def test_fully_masked_row_is_zero_and_batch_independent(t5_dirs):
    cond = _conditioner('base', t5_dirs['base'])
    W, b = cond.output_proj.weight, cond.output_proj.bias
    ids, mask = G.hand_ids(3, T=150)
    mask[0, 100:] = 0
    mask[1] = 0   # straight to the C-ABI: every key of row 1 is masked
    out, hid = cond.t5.encode(ids, mask, W, b, return_hidden=True)
    assert torch.isfinite(hid).all() and torch.isfinite(out).all()
    assert bool((out[1] == 0).all()) and bool((out[0, 100:] == 0).all())
    # item 0 alone at its own length (100 tokens, two key tiles) and inside the batch padded to 150: bit-identical
    alone, _ = cond.t5.encode(ids[:1, :100], mask[:1, :100], W, b)
    assert torch.equal(alone[0], out[0, :100]), "padding the batch changed an item's output"
    solo, _ = cond.t5.encode(ids[2:3], mask[2:3], W, b)
    assert torch.equal(solo[0], out[2]), "an item's output depends on the other items of its batch"


def test_refuses_out_of_range_ids(t5_dirs):
    cond = _conditioner('base', t5_dirs['base'])
    with pytest.raises(ValueError):
        cond.t5.encode(torch.tensor([[32128]]), torch.ones(1, 1, dtype=torch.long), cond.output_proj.weight,
                       cond.output_proj.bias)


# ----------------------------------------------------------------------------- end to end from a checkpoint directory

def _codec_pkg(name):
    import yaml
    c = synth.ENCODEC_CONFIGS[name]
    xp = dict(channels=c['channels'], sample_rate=c['sample_rate'],
              seanet=dict(dimension=c['dimension'], n_filters=c['n_filters'], n_residual_layers=c['n_residual_layers'],
                          ratios=c['ratios'], kernel_size=c['kernel_size'], last_kernel_size=c['last_kernel_size'],
                          residual_kernel_size=c['residual_kernel_size'], dilation_base=c['dilation_base'],
                          pad_mode=c['pad_mode'], compress=c['compress'], lstm=c['lstm'], norm=c['norm']),
              rvq=dict(n_q=c['n_q'], bins=c['bins']), encodec=dict(causal=c['causal'], renormalize=c['renormalize']))
    return {'best_state': synth.synth_encodec_state_dict(c, 5), 'xp.cfg': yaml.safe_dump(xp)}


def _checkpoint_dir(path, t5_name, codec, melody=False):
    """A reference-format MusicGen / AudioGen directory: state_dict.bin and compression_state_dict.bin with their xp.cfg."""
    import yaml
    base = 'lm_mini_melody' if melody else 'lm_mini'
    cfg = dict(synth.lm_config(base), cond_dim=synth.T5_CONFIGS[t5_name]['d_model'], card=2048, num_layers=2)
    fuser = dict(cross_attention_pos_emb=False, sum=[], input_interpolate=[],
                 prepend=['self_wav', 'description'] if melody else [], cross=[] if melody else ['description'])
    conds = {'description': {'model': 't5', 't5': {'name': t5_name, 'finetune': False, 'word_dropout': 0.3,
                                                   'normalize_text': False}}}
    if melody:
        conds['self_wav'] = {'model': 'chroma_stem', 'chroma_stem': dict(sample_rate=32000, n_chroma=12, radix2_exp=14,
                                                                         argmax=True, match_len_on_eval=True, eval_wavs=None,
                                                                         n_eval_wavs=0, cache_path=None)}
    xp = dict(sample_rate=synth.ENCODEC_CONFIGS[codec]['sample_rate'], dataset={'segment_duration': 1.0},
              transformer_lm=dict(dim=cfg['dim'], num_heads=cfg['num_heads'], num_layers=cfg['num_layers'], n_q=4,
                                  card=cfg['card'], norm_first=True),
              codebooks_pattern={'modeling': 'delay', 'delay': {'delays': [0, 1, 2, 3]}},
              classifier_free_guidance={'inference_coef': 3.0}, fuser=fuser, conditioners=conds)
    os.makedirs(path, exist_ok=True)
    torch.save({'best_state': synth.synth_lm_state_dict(cfg, seed=9), 'xp.cfg': yaml.safe_dump(xp)},
               os.path.join(path, 'state_dict.bin'))
    torch.save(_codec_pkg(codec), os.path.join(path, 'compression_state_dict.bin'))
    return path


DESCS = ['calm piano melody with soft strings', 'heavy techno beat', None]


def _cross_of(lm, descs):
    cond = lm.condition_provider.conditioners['description']
    return cond(cond.tokenize(list(descs) + [None] * len(descs)))[0]


@pytest.mark.parametrize('kind', ['musicgen', 'audiogen'])
def test_generate_from_local_t5(kind, tmp_path, t5_dirs):
    from audiocraft_b200.conditioners import T5Conditioner
    from audiocraft_b200.musicgen import AudioGen, MusicGen
    t5_case, t5_name, codec, cls = (('base', 't5-base', 'encodec_32k', MusicGen) if kind == 'musicgen'
                                    else ('large', 't5-large', 'encodec_16k', AudioGen))
    ckpt = _checkpoint_dir(str(tmp_path / kind), t5_name, codec)
    model = cls.get_pretrained(ckpt, text_encoder=t5_dirs[t5_case])
    assert isinstance(model.lm.condition_provider.conditioners['description'], T5Conditioner)
    model.set_generation_params(use_sampling=False, duration=0.4)
    wav, tokens = model.generate(DESCS, return_tokens=True)
    assert torch.isfinite(wav).all() and tokens.shape == (3, 4, 20)
    cross = _cross_of(model.lm, DESCS)
    assert bool((cross[3:] == 0).all()) and bool((cross[2] == 0).all())
    want = model.lm.generate(None, [], num_samples=3, max_gen_len=20, use_sampling=False, cfg_coef=3.0,
                             cross_attention_src=cross)
    assert torch.equal(tokens, want)


def test_melody_prepend_description_from_local_t5(tmp_path, t5_dirs):
    from audiocraft_b200.conditioners import T5Conditioner, identity_stem_separator
    from audiocraft_b200.musicgen import MusicGen
    ckpt = _checkpoint_dir(str(tmp_path / 'melody'), 't5-base', 'encodec_32k', melody=True)
    model = MusicGen.get_pretrained(ckpt, text_encoder=t5_dirs['base'], stem_separator=identity_stem_separator)
    lm = model.lm
    assert isinstance(lm.condition_provider.conditioners['description'], T5Conditioner)
    model.set_generation_params(use_sampling=False, duration=0.4)
    melody = torch.randn(2, 1, 32000, generator=torch.Generator().manual_seed(4)) * 0.1
    descs = DESCS[:2]
    wav, tokens = model.generate_with_chroma(descs, melody, 32000, return_tokens=True)
    assert torch.isfinite(wav).all() and tokens.shape == (2, 4, 20)
    attrs = model._prepare_tokens_and_attributes(descs, None, list(melody.cuda()))[0]
    _, prefix = lm._condition_tensors(attrs)
    desc = _cross_of(lm, descs)
    assert torch.equal(prefix[:, -desc.shape[1]:], desc), "the prefix ends with the T5 conditioner's output"
    want = lm.generate(None, [], num_samples=2, max_gen_len=20, use_sampling=False, cfg_coef=3.0, prefix=prefix)
    assert torch.equal(tokens, want)
