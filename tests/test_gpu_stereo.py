"""Stereo MusicGen on the device: 8 interleaved codebooks (`b (k c) t`, delays [0,0,1,1,2,2,3,3]) through decode, prompt prefill,
the melody prefix, scoring and the public generation surface.

At n_q = 8 and card 2048 the heads GEMM is N = 16384 wide: 1024 16-feature tiles (512 with 32-feature tiles) on
lm_gemm_kernel at rows <= 64, 256 64-feature tiles on lm_gemm_wide_kernel at rows 65-256, a sampler grid of (8, batch), a
delay write-back where two codebooks share each mask column, and 16384-wide `part` / logits rows.

Tolerances are DESIGN.md section 4's: teacher-forced CFG logits vs the fp16-emulating oracle rtol 2e-2 / atol 3e-2, vs the fp32
reference 6e-2; prefill K/V caches vs one position per step atol 4e-3, greedy tokens > 95 % equal; compute_predictions within
6e-2 of the reference; full depth CFG-mixed logits within 1.2e-1 of the fp32 reference, top-1 equal outside near-ties.  Batch
independence on the wide GEMM is exact."""
import os

import pytest
import torch

from tests import helpers as H
from tests.prefix_oracle import PrefixLMOracle
from audiocraft_b200 import synth
from oracle import lm_oracle as LO

pytestmark = pytest.mark.gpu

K = 8


def _lm(name, wseed, **over):
    from audiocraft_b200.lm import LMModel
    cfg = synth.lm_config(name)
    cfg.update(over)
    sd = synth.synth_lm_state_dict(cfg, seed=wseed)
    return cfg, sd, LMModel(sd, cfg, None, None)


def _golden(name='lm_mini_stereo.pt'):
    p = os.path.join(H.GOLDEN_DIR, name)
    if not os.path.exists(p):
        pytest.skip(f'{name} not generated')
    return torch.load(p, weights_only=False)


def _close(got, ref, rtol, atol, what):
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = (got - ref).abs()
    print(f'{what}: max err {err.max().item():.2e}, {(err / (atol + rtol * ref.abs())).max().item():.2f} of tolerance')
    torch.testing.assert_close(got, ref, rtol=rtol, atol=atol, msg=lambda m: f'{what}: {m}')


def _teacher_forced_oracle(cfg, sd, cross, B, T, seed):
    seq = torch.randint(0, cfg['card'], (B, K, T + 4), generator=torch.Generator().manual_seed(seed))
    o = LO.LMOracle(sd, cfg, half_gemm=True)
    rec = []
    o.generate(None, cross, B, T, use_sampling=False, record_logits=rec, teacher=seq)
    return o.last_sequence, torch.stack(rec)


# rows = 2B: <= 16 and 17-32 and 33-64 on lm_gemm_kernel (NT 1 / 2 / 4 / 8), 66-256 on the wide GEMM (NPAD 128 / 256)
@pytest.mark.parametrize('name,B', [
    ('lm_mini_stereo', 2), ('lm_mini_stereo', 12), ('lm_mini_stereo', 24), ('lm_mini_stereo', 33), ('lm_mini_stereo', 128),
    ('lm_medium_2l_stereo', 8), ('lm_medium_2l_stereo', 12), ('lm_medium_2l_stereo', 32), ('lm_medium_2l_stereo', 65),
    ('lm_medium_2l_stereo', 128)])
def test_teacher_forced_cfg_logits_match_fp16_oracle(name, B):
    cfg, sd, m = _lm(name, 11)
    _, _, cross = H.lm_condition(cfg, sd, B, 7, 3)
    seq, ref = _teacher_forced_oracle(cfg, sd, cross, B, 4, B)
    lg = m.teacher_forced_logits(seq, cross, cfg['cfg_coef']).cpu()
    assert lg.shape == (seq.shape[-1] - 1, B, K, cfg['card'])
    _close(lg, ref, 2e-2, 3e-2, f'{name} rows={2 * B}')


def test_ft32_tiles_equal_16_feature_tiles_at_8_codebooks(monkeypatch):
    """The N = 16384 heads GEMM on 32-feature tiles (the default at d = 1536) and on 16-feature tiles: bit-identical logits."""
    cfg, sd, m = _lm('lm_medium_2l_stereo', 7)
    _, _, cross = H.lm_condition(cfg, sd, 8, 6, 2)
    seq = torch.randint(0, cfg['card'], (8, K, 9), generator=torch.Generator().manual_seed(3))
    wide = m.teacher_forced_logits(seq, cross, 3.0).cpu()
    monkeypatch.setenv('ACB_LM_FT32', '0')
    narrow = m.teacher_forced_logits(seq, cross, 3.0).cpu()
    assert torch.isfinite(wide).all()
    assert torch.equal(wide, narrow), f'max diff {(wide - narrow).abs().max():.3e}'


def test_item_logits_do_not_depend_on_the_batch():
    """The same 33 items at B = 33 (rows 66, NPAD 128) and as the first 33 of B = 128 (rows 256, NPAD 256): every item's raw
    per-row logits, cond and null rows, are bit-identical."""
    cfg, sd, m = _lm('lm_medium_2l_stereo', 7)
    _, _, cross = H.lm_condition(cfg, sd, 128, 6, 2)
    seq = torch.randint(0, cfg['card'], (128, K, 6), generator=torch.Generator().manual_seed(1))
    _, big = m.teacher_forced_logits(seq, cross, cfg['cfg_coef'], raw=True)
    _, small = m.teacher_forced_logits(seq[:33], torch.cat([cross[:33], cross[128:161]], 0), cfg['cfg_coef'], raw=True)
    assert torch.equal(small[:, :33], big[:, :33]), 'cond rows differ between batch 33 and batch 128'
    assert torch.equal(small[:, 33:], big[:, 128:161]), 'null rows differ between batch 33 and batch 128'


def _near_tie_only(got_seq, want_seq, mixed, what, tol=6e-2):
    """Greedy tokens equal, or the first differing sequence step is a near-tie of `mixed` [S-1, B, K, card] (CFG-mixed logits
    along `want_seq`)."""
    if torch.equal(got_seq, want_seq):
        return
    step = int((got_seq != want_seq).any(0).any(0).nonzero()[0])
    top2 = mixed[step - 1].topk(2, dim=-1).values
    gap = (top2[..., 0] - top2[..., 1])[got_seq[..., step] != want_seq[..., step]]
    print(f'{what}: first divergence at sequence step {step}, top-2 gaps {gap.tolist()}')
    assert (gap < tol).all(), f'{what}: greedy token differs from the reference although its argmax margin is clear'


def test_lm_mini_stereo_matches_reference_golden():
    """Teacher-forced CFG logits along the reference's greedy sequence (6e-2), greedy generation and a greedy continuation of a
    5-frame prompt (prefilled) equal to the reference's tokens outside near-ties."""
    g = _golden()
    cfg, sd, m = _lm(g['name'], g['wseed'])
    B, T = g['batch'], g['T']
    _, _, cross = H.lm_condition(cfg, sd, B, g['t_text'], g['cseed'])
    lg = m.teacher_forced_logits(g['sequence'], cross, cfg['cfg_coef']).cpu()
    _close(lg[..., g['logits_idx']], g['logits'], 6e-2, 6e-2, 'stereo CFG logits vs fp32 reference')
    agree = lg.argmax(-1) == g['logits_argmax'].long()
    assert bool(agree[g['logits_margin'] > 6e-2].all())
    out = m.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross)
    assert out.shape == (B, K, T) and out.dtype == torch.int64
    _near_tie_only(m.last_sequence.cpu(), g['sequence'], lg, 'greedy')
    P = g['prompt_len']
    got = m.generate(g['greedy'][..., :P].cuda(), [], num_samples=B, max_gen_len=T, use_sampling=False,
                     cross_attention_src=cross).cpu()
    assert torch.equal(got[..., :P], g['greedy'][..., :P])
    want_seq = LO.build_delay_sequence(g['continuation'], cfg['delays'], cfg['card'])[0]
    _near_tie_only(m.last_sequence.cpu(), want_seq, m.teacher_forced_logits(want_seq, cross, cfg['cfg_coef']).cpu(),
                   'continuation')


@pytest.mark.parametrize('kw', [dict(top_k=10, temp=0.9), dict(top_k=0, top_p=0.8), dict(top_k=250, temp=1.0)],
                         ids=['top_k', 'top_p', 'top_k_250'])
def test_sampling_with_injected_noise_matches_oracle(kw):
    """Top-k / top-p draws over the (8, batch) sampler grid with the oracle's Exponential(1) noise: the same tokens, or a first
    divergence where the GPU's pick scores within 3 % of the oracle's best (an fp16 near-tie)."""
    cfg, sd, m = _lm('lm_mini_stereo', 3)
    B, T = 3, 10
    _, _, cross = H.lm_condition(cfg, sd, B, 5, 1)

    def nf(step, shape):
        return H.exp_noise(23, step, shape[0] * shape[1], shape[2])

    o = LO.LMOracle(sd, cfg, half_gemm=True)
    want = o.generate(None, cross, B, T, use_sampling=True, noise_fn=nf, **kw)
    m._debug_noise_fn = lambda step, shape: nf(step, shape).cuda()
    try:
        got = m.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=True, cross_attention_src=cross, **kw)
    finally:
        m._debug_noise_fn = None
    assert got.shape == (B, K, T)
    agree = (got.cpu() == want).float().mean().item()
    print(f'sampled {kw}: token agreement {agree:.3f}')
    if agree == 1.0:
        return
    gseq, oseq = m.last_sequence.cpu(), o.last_sequence
    step = int((gseq != oseq).any(0).any(0).nonzero()[0])
    rec = []
    o.generate(None, cross, B, T, use_sampling=True, noise_fn=nf, record_logits=rec, teacher=gseq, **kw)
    probs = torch.softmax(rec[step - 1] / kw.get('temp', 1.0), -1)
    noise = nf(step, (B, K, cfg['card'])).reshape(probs.shape)
    if kw.get('top_p', 0.0) > 0:
        ps, pi = LO.top_p_sorted(probs, kw['top_p'])
        score = torch.zeros_like(probs).scatter(-1, pi, ps / noise)
    else:
        score = LO.top_k_filter(probs, kw['top_k']) / noise
    valid = torch.from_numpy(LO.delay_sequence_indexes(T, K, cfg['delays'])[1][:, step])
    picked = score.gather(-1, gseq[..., step].clamp(max=cfg['card'] - 1).unsqueeze(-1)).squeeze(-1)
    rel = (picked / score.max(-1).values)[:, valid]
    print(f'   first divergence at sequence step {step}: GPU pick / oracle best score = {rel.min():.4f}')
    assert rel.min() > 0.97


@pytest.mark.parametrize('B,T0', [(5, 23), (40, 22)], ids=['rows10', 'rows80-wide'])
def test_prompt_prefill_equals_token_by_token(monkeypatch, B, T0):
    """A prompt of T0 frames at 8 codebooks, prefilled (several positions per pass at rows 10, one position of every row per pass
    on the wide GEMM at rows 80) vs one decode step per position (ACB_LM_PREFILL=0): same K / V caches, same greedy tokens."""
    cfg, sd, m = _lm('lm_mini_stereo', 5)
    T = T0 + 6
    _, _, cross = H.lm_condition(cfg, sd, B, 5, 1)
    prompt = torch.randint(0, cfg['card'], (B, K, T0), generator=torch.Generator().manual_seed(3))
    out_pf = m.generate(prompt.cuda(), [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross).cpu()
    kc_pf = m._bufs['k_cache'][:, :2 * B, :, :T0].clone()
    vc_pf = m._bufs['v_cache'][:, :2 * B, :, :T0].clone()
    monkeypatch.setenv('ACB_LM_PREFILL', '0')
    out_ss = m.generate(prompt.cuda(), [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross).cpu()
    _close(kc_pf.float(), m._bufs['k_cache'][:, :2 * B, :, :T0].float(), 0, 4e-3, f'rows={2 * B} K cache')
    _close(vc_pf.float(), m._bufs['v_cache'][:, :2 * B, :, :T0].float(), 0, 4e-3, f'rows={2 * B} V cache')
    assert torch.equal(out_pf[..., :T0], prompt)
    agree = (out_pf == out_ss).float().mean()
    print(f'token agreement {agree:.4f}')
    assert agree > 0.95


@pytest.mark.parametrize('B,P', [(2, 23), (40, 19)], ids=['rows4', 'rows80-wide'])
def test_melody_prefix_logits_match_oracle(B, P):
    """A condition prefix (MusicGen-stereo-melody's layout: no cross attention) in front of 8-codebook tokens: teacher-forced
    CFG logits vs the prefix oracle, fp16-emulating (2e-2) and fp32 (6e-2)."""
    cfg, sd, m = _lm('lm_mini_melody_stereo', 5)
    S = 16
    seq = H.fullsize_sequence(cfg, B, S - max(cfg['delays']) - 1, 4)
    prefix = torch.randn(2 * B, P, cfg['dim'], generator=torch.Generator().manual_seed(13)) * 0.5
    out = m.teacher_forced_logits(seq, None, cfg['cfg_coef'], prefix=prefix).cpu()
    for half, tol in ((True, 2e-2), (False, 6e-2)):
        ref = PrefixLMOracle(sd, cfg, half_gemm=half, prefix=prefix).teacher_forced_mixed(seq, None, cfg['cfg_coef'])
        _close(out, ref, tol, tol, f'prefix P={P} rows={2 * B} half={half}')


def test_compute_predictions_match_reference_golden():
    """LMModel.compute_predictions on stereo codes: logits [B, 8, T, 2048] within 6e-2 of the reference's, top-1 equal outside
    margins of 0.15, NaN pattern and mask equal."""
    g = _golden()
    p = g['predictions']
    cfg, sd, m = _lm(g['name'], g['wseed'])
    B = g['batch']
    cross = H.lm_condition(cfg, sd, B, g['t_text'], g['cseed'])[2][:B]
    codes = torch.randint(0, cfg['card'], (B, K, p['T']), generator=torch.Generator().manual_seed(p['kseed']))
    for key, valid in (('valid', True), ('all', False)):
        out = m.compute_predictions(codes, keep_only_valid_steps=valid, cross_attention_src=cross)
        lg = out.logits.cpu()
        assert lg.shape == (B, K, p['T'], cfg['card'])
        assert torch.equal(out.mask.cpu(), p[f'mask_{key}'][None].expand(B, -1, -1))
        assert torch.equal(torch.isnan(lg).all(-1), p[f'nan_{key}']) and torch.equal(torch.isnan(lg).any(-1), p[f'nan_{key}'])
        ok = ~p[f'nan_{key}']
        ti = p[f'top_i_{key}'].long()
        err = torch.cat([(lg.gather(-1, ti) - p[f'top_v_{key}']).abs()[ok].flatten(),
                         (lg[..., g['logits_idx']] - p[f'logits_{key}']).abs()[ok].flatten()])
        margin = (p[f'top_v_{key}'][..., 0] - p[f'top_v_{key}'][..., 1])[ok]
        agree = lg.argmax(-1)[ok] == ti[..., 0][ok]
        print(f'keep_only_valid_steps={valid}: max |logit diff| vs fp32 reference {float(err.max()):.4f}')
        assert float(err.max()) < 6e-2
        assert bool(agree[margin > 0.15].all())


def test_fulldepth_stereo_medium_logits_match_reference_cpu_golden():
    """Full-depth MusicGen-stereo-medium over a 1500-frame sequence (KV length up to 1503, rows 8): CFG-mixed logits within
    1.2e-1 of the reference's fp32 CPU forward, top-1 equal outside near-ties."""
    g = _golden('musicgen_stereo_medium_full.pt')
    name = g['name']
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=g['wseed'])
    _, _, cross = H.lm_condition(cfg, sd, g['batch'], g['t_text'], g['cseed'])
    seq = H.fullsize_sequence(cfg, g['batch'], g['T'], g['sseed'])
    assert torch.equal(seq[..., :16], g['seq_head'])
    from audiocraft_b200.lm import LMModel
    m = LMModel(sd, cfg, None, None, 'cuda')
    del sd
    S = seq.shape[-1]
    lg = m.teacher_forced_logits(seq, cross, cfg['cfg_coef'], n_steps=S - 1, keep=g['steps']).cpu()
    ti = g['logits_top_i'].long()
    err = (lg.gather(-1, ti) - g['logits_top_v']).abs()
    print(f'{name}: max |CFG-mixed logit diff| vs fp32 reference per kept step:',
          [round(float(e), 4) for e in err.amax(dim=(1, 2, 3))])
    assert float(err.max()) < 1.2e-1
    margin = g['logits_top_v'][..., 0] - g['logits_top_v'][..., 1]
    agree = lg.argmax(-1) == ti[..., 0]
    assert bool(agree[margin > 1.2e-1].all()), 'top-1 token differs from the reference outside a near-tie'


def test_stereo_codec_matches_reference_golden():
    """The interleaved stereo codec over encodec_32k: codes of a stereo input equal the reference's (except RVQ near-ties), and
    decoding the reference's codes gives its waveform."""
    from audiocraft_b200.encodec import EncodecModel, InterleaveStereoCompressionModel
    c = _golden()['codec']
    cfg = synth.ENCODEC_CONFIGS[c['name']]
    sd = synth.synth_encodec_state_dict(cfg, seed=c['wseed'])
    cm = InterleaveStereoCompressionModel(EncodecModel(sd, cfg, 'cuda'))
    assert (cm.num_codebooks, cm.frame_rate, cm.channels, cm.cardinality, cm.total_codebooks) == c['props']
    x = H.audio_input(dict(cfg, channels=2), c['codes'].shape[0], c['length'], c['xseed'])
    codes, scale = cm.encode(x.cuda())
    assert scale is None and codes.shape == c['codes'].shape
    same = codes.cpu() == c['codes']
    if not bool(same.all()):   # judge the first differing level of each (channel, frame) by the reference's own margin
        from oracle import encodec_oracle as EO
        B = x.shape[0]
        o = EO.EncodecOracle(sd, cfg)
        lat = o.encode_latent(x.transpose(0, 1).reshape(2 * B, 1, -1))
        _, margins = EO.rvq_encode(lat, EO.codebooks_of(sd, cfg['n_q']), return_margin=True)   # [2B, 4, T]
        margins = margins.view(2, B, 4, -1).permute(1, 2, 0, 3).reshape(B, 8, -1)
        neq = (~same).view(B, 4, 2, -1)
        first = (neq.int().cumsum(1).eq(1) & neq).view(B, 8, -1)
        print(f'{int(first.sum())} near-tie code flips, reference margins {margins[first].tolist()[:8]}')
        assert (margins[first].abs() < 1e-4).all(), 'RVQ index mismatch with a clear margin'
    wav = cm.decode(c['codes'].cuda(), None).cpu()
    assert wav.shape == (x.shape[0], 2, c['wav_len'])
    torch.testing.assert_close(wav[..., ::c['wav_stride']], c['wav_strided'], rtol=0, atol=1e-4)


# ----------------------------------------------------------------------------- public surface
@pytest.fixture(scope='module')
def stereo_small():
    from audiocraft_b200.musicgen import MusicGen
    return MusicGen.get_pretrained('synthetic/stereo-small')


def _decoded(mg, tok):
    """The returned tokens decoded through the model's stereo codec."""
    return mg.compression_model.decode(tok, None)


def test_stereo_generate_shapes_and_decode(stereo_small):
    mg = stereo_small
    assert (mg.audio_channels, mg.sample_rate, mg.frame_rate, mg.lm.num_codebooks) == (2, 32000, 50, 8)
    assert mg.compression_model.num_codebooks == 8
    mg.set_generation_params(duration=1.0, top_k=250)
    wav, tok = mg.generate(['stereo pads', 'wide drums'], return_tokens=True)
    assert tuple(wav.shape) == (2, 2, 32000) and tuple(tok.shape) == (2, 8, 50)
    assert torch.isfinite(wav).all() and int(tok.min()) >= 0 and int(tok.max()) < 2048
    assert torch.equal(_decoded(mg, tok), wav)
    wav, tok = mg.generate_unconditional(3, return_tokens=True)
    assert tuple(wav.shape) == (3, 2, 32000) and tuple(tok.shape) == (3, 8, 50)
    assert torch.equal(_decoded(mg, tok), wav)


def test_stereo_generate_continuation(stereo_small):
    """A 2-channel prompt is encoded through the interleaved codec and kept as the first frames; a mono prompt is turned into 2
    identical channels by convert_audio, so its left and right codes are equal."""
    mg = stereo_small
    mg.set_generation_params(duration=1.0, use_sampling=False)
    x = H.audio_input(dict(sample_rate=32000, channels=2), 2, 8000, 1)
    wav, tok = mg.generate_continuation(x, 32000, ['a', None], return_tokens=True)
    assert tuple(wav.shape) == (2, 2, 32000) and tuple(tok.shape) == (2, 8, 50)
    ptok, _ = mg.compression_model.encode(x.cuda())
    assert torch.equal(tok[..., :ptok.shape[-1]], ptok)
    assert torch.equal(_decoded(mg, tok), wav)
    mono = H.audio_input(dict(sample_rate=16000, channels=1), 1, 4000, 2)
    wav, tok = mg.generate_continuation(mono, 16000, ['a'], return_tokens=True)
    assert tuple(wav.shape) == (1, 2, 32000)
    n = 8000 * 50 // 32000   # prompt frames: 4000 samples at 16 kHz are 8000 at 32 kHz
    left, right = tok.view(1, 4, 2, -1)[..., :n].unbind(2)
    assert torch.equal(left, right)


def test_stereo_long_generation_slides_the_window(stereo_small):
    """Beyond max_duration the generation runs window by window, each prompted with the tail of the previous one, at 8
    codebooks."""
    mg = stereo_small
    saved = mg.max_duration
    mg.max_duration = 2.0
    try:
        mg.set_generation_params(duration=3.0, extend_stride=1.0, use_sampling=False)
        wav, tok = mg.generate(['long one'], return_tokens=True)
    finally:
        mg.max_duration = saved
    assert tuple(tok.shape) == (1, 8, 150) and tuple(wav.shape) == (1, 2, 96000)
    assert torch.equal(_decoded(mg, tok), wav)


def test_stereo_melody_generate_with_chroma():
    """synthetic/stereo-melody: the chroma comes from the stereo melody's channel mean, as in the reference (the wav collation
    averages channels), so a stereo melody and its mono mix give the same greedy tokens; outputs are [B, 2, T]."""
    from audiocraft_b200.musicgen import MusicGen
    mg = MusicGen.get_pretrained('synthetic/stereo-melody')
    assert mg.audio_channels == 2 and mg.lm.n_q == 8 and mg._has_melody
    mg.set_generation_params(duration=1.0, use_sampling=False)
    melody = H.audio_input(dict(sample_rate=32000, channels=2), 2, 32000, 7)
    wav, tok = mg.generate_with_chroma(['x', 'y'], melody, 32000, return_tokens=True)
    assert tuple(wav.shape) == (2, 2, 32000) and tuple(tok.shape) == (2, 8, 50)
    assert torch.equal(_decoded(mg, tok), wav)
    _, tok_mono = mg.generate_with_chroma(['x', 'y'], melody.mean(1, keepdim=True), 32000, return_tokens=True)
    assert torch.equal(tok_mono, tok)
    wav, tok = mg.generate(['x'], return_tokens=True)   # null melody
    assert tuple(wav.shape) == (1, 2, 32000) and tuple(tok.shape) == (1, 8, 50)
