"""GPU tests of the full-sequence forward (LMModel.forward / compute_predictions on acb_lm_forward).

Tolerances are DESIGN.md section 4's: logits vs the fp32 reference 6e-2; vs the fp16-emulating oracle rtol 2e-2 / atol 3e-2
(4e-2 with rotary positions: fp16 q / k after the rotation); full depth vs the reference's CUDA autocast path 5e-2 per row and
1.2e-1 for CFG-mixed rows vs the fp32 reference; top-1 equal outside margins of 0.15 (resp. 1.2e-1)."""
import os

import pytest
import torch

from tests import helpers as H
from tests.prefix_oracle import PrefixLMOracle
from audiocraft_b200 import synth
from oracle import lm_oracle as LO

pytestmark = pytest.mark.gpu


def _lm(name, wseed, **over):
    from audiocraft_b200.lm import LMModel
    cfg = synth.lm_config(name)
    cfg.update(over)
    sd = synth.synth_lm_state_dict(cfg, seed=wseed)
    return cfg, sd, LMModel(sd, cfg, None, None)


def _golden(name):
    p = os.path.join(H.GOLDEN_DIR, name)
    if not os.path.exists(p):
        pytest.skip(f'{name} not generated')
    return torch.load(p, weights_only=False)


def _random_seq(cfg, B, S, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, cfg['card'] + 1, (B, cfg['n_q'], S), generator=g)   # codes and the special token


@pytest.mark.parametrize('name', ['lm_tiny', 'lm_mini', 'musicgen_small'])
def test_compute_predictions_match_reference_golden(name):
    case = _golden('lm_predictions.pt')['cases'][name]
    cfg, sd, m = _lm(name, case['wseed'])
    B, T = case['batch'], case['T']
    cross = H.lm_condition(cfg, sd, B, case['t_text'], case['cseed'])[2][:B]   # the condition rows, no CFG
    codes = torch.randint(0, cfg['card'], (B, cfg['n_q'], T), generator=torch.Generator().manual_seed(case['kseed']))
    for key, valid in (('valid', True), ('all', False)):
        out = m.compute_predictions(codes, keep_only_valid_steps=valid, cross_attention_src=cross)
        lg = out.logits.cpu()
        assert torch.equal(out.mask.cpu(), case[f'mask_{key}'][None].expand(B, -1, -1))
        assert torch.equal(torch.isnan(lg).all(-1), case[f'nan_{key}']) and torch.equal(torch.isnan(lg).any(-1), case[f'nan_{key}'])
        ok = ~case[f'nan_{key}']
        if case['topn'] is None:
            want = case[f'logits_{key}']
            err = (lg - want).abs()[ok]
            top2 = want[ok].topk(2, dim=-1).values
            margin, agree = top2[:, 0] - top2[:, 1], lg[ok].argmax(-1) == want[ok].argmax(-1)
        else:
            ti = case[f'top_i_{key}'].long()
            got = lg.gather(-1, ti)
            err = (got - case[f'top_v_{key}']).abs()[ok]
            margin = (case[f'top_v_{key}'][..., 0] - case[f'top_v_{key}'][..., 1])[ok]
            agree = lg.argmax(-1)[ok] == ti[..., 0][ok]
        print(f'{name} keep_only_valid_steps={valid}: max |logit diff| vs fp32 reference {float(err.max()):.4f}')
        assert float(err.max()) < 6e-2
        assert bool(agree[margin > 0.15].all())


# d = 192, ffn = int(4.25 * 192) = 816, card = 100: every GEMM but the cross K/V one (N = 2d = 384) has a ragged N tile
# (3d = 576, d = 192, ffn = 816, n_q * card = 400 against 128-wide tiles), and linear2 a ragged K tile (816 = 12 * 64 + 48)
RAGGED = dict(dim=192, num_heads=3, hidden_scale=4.25, card=100)


@pytest.mark.parametrize('name,B,S,text_len,pe,over', [
    ('lm_mini', 2, 37, 7, 'sin', {}), ('lm_mini', 1, 1, 1, 'sin', {}), ('lm_mini', 3, 130, 33, 'sin', {}),
    ('lm_mini', 2, 300, 77, 'sin', {}), ('lm_tiny', 3, 65, 7, 'sin', {}),
    ('lm_mini', 2, 70, 7, 'rope', {}), ('lm_mini', 2, 70, 7, 'sin_rope', {}),
    ('lm_mini', 2, 93, 11, 'sin', RAGGED), ('lm_mini', 1, 129, 33, 'rope', RAGGED),
    ('lm_medium_2l', 2, 129, 16, 'sin', {}), ('lm_large_2l', 1, 100, 9, 'sin', {}), ('musicgen_small', 2, 41, 7, 'sin', {})],
    ids=lambda v: 'ragged' if v is RAGGED else None)
def test_forward_matches_fp16_oracle(name, B, S, text_len, pe, over):
    """M tails: B * S and the text rows are off the 128-row grid in most cases.  N and K tails: the RAGGED cases (every other
    config has N and K on the tile grid)."""
    cfg, sd, m = _lm(name, 21, positional_embedding=pe, **over)
    if over:
        d, ffn = cfg['dim'], int(cfg['hidden_scale'] * cfg['dim'])
        assert (3 * d) % 128 and d % 128 and ffn % 128 and ffn % 64 and (cfg['n_q'] * cfg['card']) % 128
    cross = H.lm_condition(cfg, sd, B, text_len, 22)[2][:B]
    seq = _random_seq(cfg, B, S, 23)
    got = m.forward(seq, cross_attention_src=cross).cpu()
    want = LO.LMOracle(sd, cfg, half_gemm=True).forward(seq, cross)
    atol = 3e-2 if pe == 'sin' else 4e-2
    print(f'{name} B={B} S={S} text={text_len} {pe}: max |diff| {float((got - want).abs().max()):.4f}')
    torch.testing.assert_close(got, want, rtol=2e-2, atol=atol)


def test_forward_with_text_conditions_goes_through_provider_and_fuser():
    """`conditions` / `condition_tensors` reach the transformer through condition_provider and fuser with one row per item
    (no CFG rows, as the reference's forward); the cross source is output_proj(hidden) * mask of the text encoder."""
    from audiocraft_b200.conditioners import ConditionFuser, ConditioningAttributes, ConditioningProvider, \
        PrecomputedTextConditioner
    from audiocraft_b200.lm import LMModel
    from audiocraft_b200.loaders import synthetic_text_encoder
    cfg = synth.lm_config('lm_mini')
    sd = synth.synth_lm_state_dict(cfg, seed=81)
    enc = synthetic_text_encoder(cfg, t_text=9)
    prov = ConditioningProvider({'description': PrecomputedTextConditioner(cfg['cond_dim'], cfg['dim'], enc)})
    m = LMModel(sd, cfg, prov, ConditionFuser({'cross': ['description']}))
    texts = ['warm analog synth pads', 'drums']
    conds = [ConditioningAttributes(text={'description': t}) for t in texts]
    B, T = len(texts), 25
    codes = torch.randint(0, cfg['card'], (B, cfg['n_q'], T), generator=torch.Generator().manual_seed(82))
    seq = _random_seq(cfg, B, 26, 83)
    got = m.forward(seq, conds)
    assert got.shape == (B, cfg['n_q'], 26, cfg['card'])
    hid, mask = enc(texts)
    w = sd['condition_provider.conditioners.description.output_proj.weight']
    bias = sd['condition_provider.conditioners.description.output_proj.bias']
    cross = (hid @ w.t() + bias) * mask.unsqueeze(-1)
    want = LO.LMOracle(sd, cfg, half_gemm=True).forward(seq, cross)
    torch.testing.assert_close(got.cpu(), want, rtol=2e-2, atol=3e-2)
    # condition_tensors and conditions are the same path; compute_predictions passes them through
    tensors = m.condition_provider(m.condition_provider.tokenize(conds))
    assert torch.equal(m.forward(seq, condition_tensors=tensors), got)
    a = m.compute_predictions(codes, conds)
    b = m.compute_predictions(codes, condition_tensors=tensors)
    assert torch.equal(torch.nan_to_num(a.logits), torch.nan_to_num(b.logits)) and torch.equal(a.mask, b.mask)
    with pytest.raises(AssertionError):
        m.forward(seq, conds, condition_tensors=tensors)
    with pytest.raises(ValueError):
        m.forward(seq, conds, cross_attention_src=cross)
    with pytest.raises(ValueError):
        m.compute_predictions(codes, condition_tensors=tensors, cross_attention_src=cross)


@pytest.mark.parametrize('B,P,S', [(2, 9, 30), (1, 150, 5)])
def test_forward_with_melody_prefix_matches_oracle(B, P, S):
    cfg, sd, m = _lm('lm_mini_melody', 31)
    prefix = torch.randn(B, P, cfg['dim'], generator=torch.Generator().manual_seed(32)) * 0.5
    seq = _random_seq(cfg, B, S, 33)
    got = m.forward(seq, prefix=prefix).cpu()
    want = PrefixLMOracle(sd, cfg, half_gemm=True, prefix=prefix).forward(seq, None)
    assert got.shape == (B, cfg['n_q'], S, cfg['card'])
    torch.testing.assert_close(got, want, rtol=2e-2, atol=3e-2)


@pytest.mark.parametrize('name,batch', [('musicgen_medium', 8), ('musicgen_large', 32)])
def test_fulldepth_forward_matches_reference(name, batch):
    """The benchmarked size: 2 * batch rows ([cond; null]) x 1503 positions, against the reference's CUDA autocast forward
    (per row) and its fp32 CPU forward (CFG-mixed); for medium also against the decode path on the same sequence
    (streaming equals batch, the reference's test_transformer.py:39-49 property)."""
    g = _golden(f'{name}_cuda.pt')
    gf = _golden(f'{name}_full.pt')
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=g['wseed'], device='cuda', dtype=torch.float16)
    cross = H.lm_condition(cfg, sd, batch, g['t_text'], g['cseed'])[2].cuda()
    seq = H.fullsize_sequence(cfg, batch, g['T'], g['sseed']).cuda()
    from audiocraft_b200.lm import LMModel
    m = LMModel(sd, cfg, None, None, 'cuda')
    del sd
    S = seq.shape[-1]
    rows = 2 * batch
    lg = m.forward(torch.cat([seq, seq])[..., :S - 1], cross_attention_src=cross)    # [rows, K, S - 1, card]
    keep = torch.as_tensor(g['steps'])
    raw = lg[:, :, keep.cuda()].permute(2, 0, 1, 3)                                   # [n, rows, K, card]
    err = (raw.cpu()[..., g['index']] - g['logits'].float()).abs()
    print(f'{name} rows={rows}: max |per-row logit diff| vs reference CUDA autocast {float(err.max()):.4f}')
    assert float(err.max()) < 5e-2
    mixed = raw[:, batch:] + (raw[:, :batch] - raw[:, batch:]) * cfg['cfg_coef']
    agree = mixed.argmax(-1).cpu() == g['mix_argmax'].long()
    assert bool(agree[g['mix_margin'] > 0.15].all())
    if name == 'musicgen_medium':
        _, tf_raw = m.teacher_forced_logits(seq, cross, cfg['cfg_coef'], n_steps=S - 1, keep=g['steps'], raw=True)
        d = (tf_raw - raw).abs()
        print(f'   forward vs decode path: max |diff| {float(d.max()):.4f}')
        assert float(d.max()) < 5e-2
        top2 = tf_raw.topk(2, dim=-1).values
        agree = tf_raw.argmax(-1) == raw.argmax(-1)
        assert bool(agree[(top2[..., 0] - top2[..., 1]) > 0.15].all())


@pytest.mark.parametrize('name', ['musicgen_medium', 'musicgen_large'])
def test_fulldepth_forward_matches_reference_cpu_golden(name):
    """Full depth, 1503 positions: the CFG mix of the forward's [cond; null] rows against the reference's fp32 CPU forward
    (the weights that golden was made with come from the CPU generator)."""
    g = _golden(f'{name}_full.pt')
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=g['wseed'])
    cross = H.lm_condition(cfg, sd, g['batch'], g['t_text'], g['cseed'])[2]
    seq = H.fullsize_sequence(cfg, g['batch'], g['T'], g['sseed'])
    assert torch.equal(seq[..., :16], g['seq_head'])
    from audiocraft_b200.lm import LMModel
    m = LMModel(sd, cfg, None, None, 'cuda')
    del sd
    B, S = g['batch'], seq.shape[-1]
    lg = m.forward(torch.cat([seq, seq])[..., :S - 1], cross_attention_src=cross)
    raw = lg[:, :, torch.as_tensor(g['steps']).cuda()].permute(2, 0, 1, 3)
    mixed = (raw[:, B:] + (raw[:, :B] - raw[:, B:]) * cfg['cfg_coef']).cpu()
    ti = g['logits_top_i'].long()
    err = (mixed.gather(-1, ti) - g['logits_top_v']).abs()
    print(f'{name}: CFG-mixed forward logits vs fp32 reference: max |diff| {float(err.max()):.4f}')
    assert float(err.max()) < 1.2e-1
    margin = g['logits_top_v'][..., 0] - g['logits_top_v'][..., 1]
    assert bool((mixed.argmax(-1) == ti[..., 0])[margin > 1.2e-1].all())


@pytest.mark.parametrize('name', ['lm_mini', 'lm_medium_2l'])
def test_item_logits_are_batch_independent(name):
    cfg, sd, m = _lm(name, 41)
    B, S = 8, 77
    cross = H.lm_condition(cfg, sd, B, 11, 42)[2][:B]
    seq = _random_seq(cfg, B, S, 43)
    full = m.forward(seq, cross_attention_src=cross)
    for i in (0, 5):
        alone = m.forward(seq[i:i + 1], cross_attention_src=cross[i:i + 1])
        assert torch.equal(alone[0], full[i]), i


def test_forward_between_streaming_steps_leaves_the_stream_unchanged():
    cfg, sd, m = _lm('lm_mini', 51)
    B = 2
    cross = H.lm_condition(cfg, sd, B, 7, 52)[2]
    cols = _random_seq(cfg, B, 12, 53)

    def run(interleave):
        m.streaming_begin(B, cross, max_len=12, cfg_coef=3.0)
        outs = []
        for t in range(12):
            outs.append(m.streaming_step(cols[..., t].cuda()).clone())
            if interleave and t in (3, 7):
                m.forward(_random_seq(cfg, 3, 40, 54 + t), cross_attention_src=cross[:1].expand(3, -1, -1))
        return torch.stack(outs)
    assert torch.equal(run(False), run(True))


def test_greedy_generation_is_the_argmax_of_compute_predictions():
    cfg, sd, m = _lm('lm_mini', 61)
    B, T = 2, 30
    cross = H.lm_condition(cfg, sd, B, 7, 62)[2][:B]   # condition rows only: generate without CFG
    codes = m.generate(None, num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross)
    out = m.compute_predictions(codes, cross_attention_src=cross)
    valid = out.mask   # keep_only_valid_steps: the last max_delay timesteps of the later codebooks have no prediction
    assert float(valid.float().mean()) > 0.8
    lg = torch.nan_to_num(out.logits, nan=0.0)
    top2 = lg.topk(2, dim=-1).values
    clear = ((top2[..., 0] - top2[..., 1]) > 0.15) & valid
    assert bool((lg.argmax(-1) == codes)[clear].all())
    assert float(clear.float().sum() / valid.float().sum()) > 0.5


def test_out_of_range_tokens_raise():
    cfg, sd, m = _lm('lm_mini', 71)
    cross = H.lm_condition(cfg, sd, 1, 3, 72)[2][:1]
    seq = _random_seq(cfg, 1, 5, 73)
    seq[0, 1, 2] = cfg['card'] + 1
    with pytest.raises(IndexError):
        m.forward(seq, cross_attention_src=cross)
