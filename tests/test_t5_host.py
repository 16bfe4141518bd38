"""T5 text encoder, host side (no GPU): reading a local HF-layout directory in both weight formats, key mapping, config
parsing, the refusals, the relative-position buckets against transformers, and the tokenizer path against the golden."""
import os

import pytest
import torch

from audiocraft_b200 import loaders, synth
from audiocraft_b200 import t5 as T5
from tests import t5_golden as G

os.environ.setdefault('HF_HUB_OFFLINE', '1')


def _small_cfg(**over):
    cfg = synth.t5_config('t5-small')
    cfg.update(num_layers=2, vocab_size=300)
    cfg.update(over)
    return cfg


@pytest.mark.parametrize('fmt', ['safetensors', 'bin'])
def test_read_directory_and_map_keys(tmp_path, fmt):
    cfg = _small_cfg()
    sd = synth.synth_t5_state_dict(cfg, seed=1)
    synth.write_t5_dir(str(tmp_path), cfg, sd, G.SPIECE, fmt=fmt)
    assert os.path.exists(tmp_path / ('model.safetensors' if fmt == 'safetensors' else 'pytorch_model.bin'))
    c = T5.read_config(str(tmp_path))
    assert c == dict(d_model=512, d_kv=64, num_heads=8, num_layers=2, d_ff=2048, vocab_size=300, num_buckets=32,
                     max_distance=128, eps=1e-6)
    w = T5.map_weights(T5.read_state_dict(str(tmp_path)), c)
    blk = 'encoder.block.1.layer.'
    assert torch.equal(w['shared'], sd['shared.weight'])
    assert torch.equal(w['w_qkv'][1], torch.cat([sd[blk + f'0.SelfAttention.{n}.weight'] for n in 'qkv']))
    assert torch.equal(w['w_o'][1], sd[blk + '0.SelfAttention.o.weight'])
    assert torch.equal(w['w_i'][1], sd[blk + '1.DenseReluDense.wi.weight'])
    assert torch.equal(w['w_fo'][1], sd[blk + '1.DenseReluDense.wo.weight'])
    assert torch.equal(w['ln'][1, 1], sd[blk + '1.layer_norm.weight'])
    assert torch.equal(w['rel_bias'], sd['encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight'])
    assert torch.equal(w['final_ln'], sd['encoder.final_layer_norm.weight'])
    del sd['encoder.block.1.layer.1.DenseReluDense.wo.weight']
    with pytest.raises(KeyError):
        T5.map_weights(sd, c)


def test_synth_init_scales():
    cfg = _small_cfg()
    sd = synth.synth_t5_state_dict(cfg, seed=2)
    a = 'encoder.block.0.layer.0.SelfAttention.'
    assert abs(sd[a + 'q.weight'].std().item() - (512 * 64) ** -0.5) < 2e-4
    assert abs(sd[a + 'k.weight'].std().item() - 512 ** -0.5) < 1e-3
    assert abs(sd['encoder.block.0.layer.1.DenseReluDense.wo.weight'].std().item() - 2048 ** -0.5) < 1e-3


@pytest.mark.parametrize('over', [dict(feed_forward_proj='gated-gelu'), dict(d_kv=128, num_heads=4)])
def test_config_refusals(tmp_path, over):
    cfg = _small_cfg(**over)
    synth.write_t5_dir(str(tmp_path), cfg, {'x': torch.zeros(1)}, G.SPIECE)
    with pytest.raises(NotImplementedError):
        T5.read_config(str(tmp_path))


@pytest.mark.parametrize('kw', [dict(finetune=True), dict(normalize_text=True)])
def test_conditioner_refusals(kw):
    from audiocraft_b200.conditioners import T5Conditioner
    with pytest.raises(NotImplementedError):
        T5Conditioner('/nonexistent', 16, device='cpu', **kw)


def test_loader_refuses_d_model_mismatch(tmp_path):
    import yaml
    t5_dir = str(tmp_path / 't5')
    synth.write_t5_dir(t5_dir, _small_cfg(), {'x': torch.zeros(1)}, G.SPIECE)   # d_model 512
    xp = dict(transformer_lm=dict(dim=64, num_heads=1, num_layers=1, n_q=4, card=32, norm_first=True),
              codebooks_pattern={'modeling': 'delay', 'delay': {'delays': [0, 1, 2, 3]}},
              classifier_free_guidance={'inference_coef': 3.0}, fuser={'cross': ['description']},
              conditioners={'description': {'model': 't5', 't5': {'name': 't5-base'}}})
    path = tmp_path / 'state_dict.bin'
    torch.save({'best_state': {}, 'xp.cfg': yaml.safe_dump(xp)}, str(path))
    with pytest.raises(ValueError, match='d_model 512'):
        loaders.load_lm_model(str(path), device='cpu', text_encoder=t5_dir)
    with pytest.raises(FileNotFoundError):
        loaders.load_lm_model(str(path), device='cpu', text_encoder=str(tmp_path / 'no_such_dir'))


def test_buckets_equal_transformers():
    tr = pytest.importorskip('transformers.models.t5.modeling_t5')
    for T in (1, 2, 7, 16, 64, 129, 300, 600):
        for nb, md in ((32, 128), (16, 64)):
            got = T5.relative_position_buckets(T, nb, md)
            ctx = torch.arange(T)[:, None]
            rel = torch.arange(T)[None, :] - ctx
            want = tr.T5Attention._relative_position_bucket(rel, bidirectional=True, num_buckets=nb, max_distance=md)
            assert got.dtype == torch.int32
            assert torch.equal(got[rel + T - 1].long(), want), (T, nb, md)


def test_tokenizer_matches_golden(tmp_path):
    pytest.importorskip('transformers')
    import shutil
    shutil.copyfile(G.SPIECE, tmp_path / 'spiece.model')
    tok = T5.load_tokenizer(str(tmp_path))
    golden = torch.load(G.GOLDEN, weights_only=True)['cases']
    from audiocraft_b200.conditioners import T5Conditioner
    for name, g in golden.items():
        cond = T5Conditioner.__new__(T5Conditioner)   # tokenize only: no device encoder
        cond.t5_tokenizer = tok
        inputs = T5Conditioner.tokenize(cond, g['descs'] + [None] * len(g['descs']))
        assert torch.equal(inputs['input_ids'], g['ids']) and torch.equal(inputs['attention_mask'], g['mask']), name
        empty = [i for i, d in enumerate(g['descs'] + [None] * len(g['descs'])) if not d]
        assert bool((g['mask'][empty] == 0).all())
    assert golden['base']['ids'].shape[1] > 128   # the long prompt crosses the 64-key tiles and max_distance
