"""LM decode at 65-256 rows (33-128 CFG items per GPU), where every GEMM of the step but the cross K/V projection runs on the
wgmma kernel lm_gemm_wide_kernel (one 64-feature x all-rows tile per CTA, NPAD = 128 or 256).

Tolerances are the LM policy of tests/test_gpu_edges.py and tests/test_gpu_lm.py: teacher-forced logits vs the fp16-emulating
oracle rtol 2e-2 / atol 3e-2 (4e-2 with rotary positions); prefill K/V caches vs one position per step atol 4e-3 and greedy
tokens > 95 % equal; per-row logits vs the reference's CUDA autocast path atol 5e-2.  Batch independence is exact: the wide
GEMM's K split depends on (N, K, SM count) only."""
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


def _close(got, ref, rtol, atol, what):
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = (got - ref).abs()
    print(f'{what}: max err {err.max().item():.2e}, {(err / (atol + rtol * ref.abs())).max().item():.2f} of tolerance')
    torch.testing.assert_close(got, ref, rtol=rtol, atol=atol, msg=lambda m: f'{what}: {m}')


def _teacher_forced_oracle(cfg, sd, cross, B, T, seed):
    seq = torch.randint(0, cfg['card'], (B, 4, T + 4), generator=torch.Generator().manual_seed(seed))
    o = LO.LMOracle(sd, cfg, half_gemm=True)
    rec = []
    o.generate(None, cross, B, T, use_sampling=False, record_logits=rec, teacher=seq)
    return o.last_sequence, torch.stack(rec)


# rows = 2B; ragged row counts (66, 130) next to full tiles (128, 192 of 256, 256)
@pytest.mark.parametrize('name,B,pe', [
    ('lm_mini', 33, 'sin'), ('lm_mini', 64, 'sin'), ('lm_mini', 128, 'sin'),
    ('lm_medium_2l', 33, 'sin'), ('lm_medium_2l', 65, 'sin'), ('lm_medium_2l', 96, 'sin'), ('lm_medium_2l', 128, 'sin'),
    ('lm_medium_2l', 33, 'rope'), ('lm_medium_2l', 65, 'rope'), ('lm_medium_2l', 96, 'rope'), ('lm_medium_2l', 128, 'rope'),
    ('lm_large_2l', 65, 'sin')])
def test_wide_rows_match_oracle(name, B, pe):
    cfg, sd, m = _lm(name, 11, positional_embedding=pe)
    _, _, cross = H.lm_condition(cfg, sd, B, 7, 3)
    seq, ref = _teacher_forced_oracle(cfg, sd, cross, B, 4, B)
    lg = m.teacher_forced_logits(seq, cross, cfg['cfg_coef']).cpu()
    _close(lg, ref, 2e-2, 4e-2 if pe != 'sin' else 3e-2, f'{name} {pe} rows={2 * B}')


def test_double_cfg_rows_99_match_oracle():
    """cfg_coef_beta with [cond; style-only; null] rows at B = 33: 99 rows on the NPAD = 128 tile, streaming steps."""
    B = 33
    cfg, sd, m = _lm('lm_mini', 3)
    _, _, cross2 = H.lm_condition(cfg, sd, B, 5, 1)
    _, _, other = H.lm_condition(cfg, sd, B, 5, 4)
    cross3 = torch.cat([cross2[:B], other[:B] * 0.5, cross2[B:]], 0)
    o = LO.LMOracle(sd, cfg, half_gemm=True)
    cur = torch.full((B, cfg['n_q'], 1), cfg['card'], dtype=torch.long)
    o.reset()
    m.streaming_begin(B, cross3, max_len=10, cfg_coef=2.0, cfg_coef_beta=3.0)
    for i in range(6):
        tok, lg = o.next_token(cur, cross3, False, 1.0, 0, 0.0, 2.0, None, None, return_logits=True, cfg_coef_beta=3.0)
        got = m.streaming_step(cur[..., 0]).cpu()
        _close(got, lg, 3e-2, 3e-2, f'double CFG rows={3 * B} step {i}')
        cur = tok


def test_item_logits_do_not_depend_on_the_batch():
    """The same 33 items at B = 33 (rows 66, NPAD 128) and as the first 33 of B = 128 (rows 256, NPAD 256): every item's raw
    per-row logits, cond and null rows, are bit-identical."""
    cfg, sd, m = _lm('lm_medium_2l', 7)
    _, _, cross = H.lm_condition(cfg, sd, 128, 6, 2)
    seq = torch.randint(0, cfg['card'], (128, 4, 6), generator=torch.Generator().manual_seed(1))
    _, big = m.teacher_forced_logits(seq, cross, cfg['cfg_coef'], raw=True)
    small_cross = torch.cat([cross[:33], cross[128:161]], 0)
    _, small = m.teacher_forced_logits(seq[:33], small_cross, cfg['cfg_coef'], raw=True)
    assert torch.equal(small[:, :33], big[:, :33]), 'cond rows differ between batch 33 and batch 128'
    assert torch.equal(small[:, 33:], big[:, 128:161]), 'null rows differ between batch 33 and batch 128'


@pytest.mark.parametrize('pe', ['sin', 'rope'])
def test_prompt_prefill_at_80_rows_equals_token_by_token(monkeypatch, pe):
    """B = 40 (rows 80): one prompt position of every row per prefill pass on the wide GEMM.  Same KV cache and greedy tokens
    as token-by-token decoding (ACB_LM_PREFILL=0)."""
    B, T0 = 40, 22
    cfg, sd, m = _lm('lm_mini', 5, positional_embedding=pe)
    T = T0 + 6
    _, _, cross = H.lm_condition(cfg, sd, B, 5, 1)
    prompt = torch.randint(0, cfg['card'], (B, 4, T0), generator=torch.Generator().manual_seed(3))
    out_pf = m.generate(prompt.cuda(), [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross).cpu()
    kc_pf = m._bufs['k_cache'][:, :2 * B, :, :T0].clone()
    vc_pf = m._bufs['v_cache'][:, :2 * B, :, :T0].clone()
    monkeypatch.setenv('ACB_LM_PREFILL', '0')
    out_ss = m.generate(prompt.cuda(), [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross).cpu()
    _close(kc_pf.float(), m._bufs['k_cache'][:, :2 * B, :, :T0].float(), 0, 4e-3, f'{pe} K cache')
    _close(vc_pf.float(), m._bufs['v_cache'][:, :2 * B, :, :T0].float(), 0, 4e-3, f'{pe} V cache')
    assert torch.equal(out_pf[..., :T0], prompt)
    agree = (out_pf == out_ss).float().mean()
    print(f'token agreement {agree:.4f}')
    assert agree > 0.95


def test_melody_prefix_at_80_rows_matches_oracle():
    """A condition prefix (no cross attention) at B = 40, rows 80: teacher-forced CFG logits vs the prefix oracle, fp16-emulating
    (2e-2) and fp32 (6e-2), the tolerances of tests/test_gpu_melody.py."""
    B, P, S = 40, 19, 16
    cfg, sd, m = _lm('lm_mini_melody', 5)
    seq = H.fullsize_sequence(cfg, B, S - max(cfg['delays']) - 1, 4)
    prefix = torch.randn(2 * B, P, cfg['dim'], generator=torch.Generator().manual_seed(13)) * 0.5
    out = m.teacher_forced_logits(seq, None, cfg['cfg_coef'], prefix=prefix).cpu()
    for half, tol in ((True, 2e-2), (False, 6e-2)):
        ref = PrefixLMOracle(sd, cfg, half_gemm=half, prefix=prefix).teacher_forced_mixed(seq, None, cfg['cfg_coef'])
        _close(out, ref, tol, tol, f'prefix P={P} rows={2 * B} half={half}')


def test_fulldepth_medium_at_80_rows_matches_reference_cuda_autocast():
    """MusicGen-medium at full depth, S = 1504, with the 8 items of the reference CUDA golden tiled 5x to B = 40 (rows 80:
    the 40 cond rows, then the 40 null rows).  Needs about 40 GB of device memory (36 GB of KV cache).  Every copy's per-row
    logits are within 5e-2 of the reference's CUDA autocast path, greedy tokens agree outside near-ties, and the 5 copies of
    each item are bit-identical."""
    path = os.path.join(H.GOLDEN_DIR, 'musicgen_medium_cuda.pt')
    g = torch.load(path, weights_only=False)
    name, b0, n = 'musicgen_medium', g['batch'], 5
    from audiocraft_b200.lm import LMModel
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=g['wseed'], device='cuda', dtype=torch.float16)
    cross8 = H.lm_condition(cfg, sd, b0, g['t_text'], g['cseed'])[2].cuda()
    cross = torch.cat([cross8[:b0]] * n + [cross8[b0:]] * n, 0)
    seq = H.fullsize_sequence(cfg, b0, g['T'], g['sseed']).cuda().repeat(n, 1, 1)
    S = seq.shape[-1]
    m = LMModel(sd, cfg, None, None, 'cuda')
    del sd
    mixed, raw = m.teacher_forced_logits(seq, cross, cfg['cfg_coef'], n_steps=S - 1, keep=g['steps'], raw=True)
    mixed, raw = mixed.cpu(), raw.cpu()
    rows = [i for _ in range(n) for i in range(b0)] + [b0 + i for _ in range(n) for i in range(b0)]
    err = (raw[..., g['index']] - g['logits'].float()[:, rows]).abs()
    print(f'rows={2 * b0 * n}: max |per-row logit diff| per kept step:', [round(float(e), 4) for e in err.amax(dim=(1, 2, 3))])
    assert float(err.max()) < 5e-2
    margin = g['mix_margin'].repeat(1, n, 1)
    agree = mixed.argmax(-1) == g['mix_argmax'].long().repeat(1, n, 1)
    print(f'greedy agreement {agree.float().mean():.4f}, outside near-ties {agree[margin > 0.15].float().mean():.4f}')
    assert bool(agree[margin > 0.15].all())
    for c in range(1, n):
        assert torch.equal(raw[:, c * b0:(c + 1) * b0], raw[:, :b0]), f'cond rows of copy {c} differ from copy 0'
        nb = n * b0
        assert torch.equal(raw[:, nb + c * b0:nb + (c + 1) * b0], raw[:, nb:nb + b0]), f'null rows of copy {c} differ'
        assert torch.equal(mixed[:, c * b0:(c + 1) * b0], mixed[:, :b0])


def test_musicgen_generate_40_descriptions():
    """MusicGen.generate with 40 descriptions (rows 80) returns [40, 1, 32000] at 1 s, and its greedy tokens equal those of
    two calls of 20 items (rows 40, the mma.sync GEMM) up to a first divergence at an fp16 near-tie."""
    from audiocraft_b200.musicgen import MusicGen
    mg = MusicGen.get_pretrained('synthetic/small')
    mg.set_generation_params(use_sampling=False, duration=1.0)
    styles = [(g, inst) for g in ('ambient', 'rock', 'jazz', 'techno', 'folk')
              for inst in ('piano', 'drums', 'strings', 'synth', 'bass', 'guitar', 'flute', 'choir')]
    descs = [f'{g} track number {i} with {inst}' for i, (g, inst) in enumerate(styles)]
    assert len(descs) == 40
    wav, tok = mg.generate(descs, return_tokens=True)
    assert tuple(wav.shape) == (40, 1, 32000)
    seq40 = mg.lm.last_sequence.cpu()
    for h in range(2):
        part = descs[20 * h:20 * (h + 1)]
        _, tok_h = mg.generate(part, return_tokens=True)
        seq_h = mg.lm.last_sequence.cpu()
        if torch.equal(tok_h.cpu(), tok[20 * h:20 * (h + 1)].cpu()):
            continue
        # only the first differing sequence step is comparable: the 20-item run's top-2 gap there must be an fp16 near-tie
        mine = seq40[20 * h:20 * (h + 1)]
        step = int((mine != seq_h).any(0).any(0).nonzero()[0])
        attrs, _ = mg._prepare_tokens_and_attributes(part, None)
        cross = mg.lm._condition_tensors(attrs)[0]
        lg = mg.lm.teacher_forced_logits(seq_h, cross, mg.generation_params['cfg_coef'], n_steps=step).cpu()
        top2 = lg[step - 1].topk(2, dim=-1).values
        gap = (top2[..., 0] - top2[..., 1])[mine[..., step] != seq_h[..., step]]
        print(f'half {h}: tokens diverge at sequence step {step}, top-2 gaps {gap.tolist()}')
        assert (gap < 5e-2).all(), 'greedy token differs from the 20-item run although its argmax margin is clear'
