"""GPU parity: MusicGen LM decode kernels vs the CPU oracle and the reference golden vectors.
Tolerances: token ids exact for the sampler on identical probabilities/noise; logits vs the fp16-emulating oracle
(same rounding points: fp16 weights + fp16 GEMM inputs, fp32 accumulate) atol/rtol 2e-2; vs the fp32 reference golden
logits atol 6e-2 (fp16 weights, the reference's own GPU dtype)."""
import os

import pytest
import torch

from tests import helpers as H
from audiocraft_b200 import synth
from oracle import lm_oracle as LO

pytestmark = pytest.mark.gpu


def _golden(name):
    return torch.load(os.path.join(H.GOLDEN_DIR, f'{name}.pt'), weights_only=False)


def _model(name, wseed):
    from audiocraft_b200.lm import LMModel
    cfg = synth.lm_config(name)
    sd = synth.synth_lm_state_dict(cfg, seed=wseed)
    return cfg, sd, LMModel(sd, cfg, None, None)


@pytest.mark.parametrize('mode', ['greedy', 'top_k', 'top_p', 'plain', 'top_k_nocfg'])
def test_sampler_matches_oracle(mode):
    from audiocraft_b200 import _lib
    import ctypes as C
    L = _lib.lib()
    B, K, card = 5, 4, 2048
    g = torch.Generator().manual_seed(7)
    cfgmix = mode != 'top_k_nocfg'
    rows = 2 * B if cfgmix else B
    logits = torch.randn(rows, K, card, generator=g) * 2.0
    noise = torch.empty(B * K, card).exponential_(1, generator=g)
    kw = dict(greedy=dict(use_sampling=False, temp=1.0, top_k=0, top_p=0.0),
              top_k=dict(use_sampling=True, temp=0.8, top_k=250, top_p=0.0),
              top_p=dict(use_sampling=True, temp=1.1, top_k=0, top_p=0.9),
              plain=dict(use_sampling=True, temp=1.0, top_k=0, top_p=0.0),
              top_k_nocfg=dict(use_sampling=True, temp=1.0, top_k=50, top_p=0.0))[mode]
    mixed = logits[B:] + (logits[:B] - logits[B:]) * 3.0 if cfgmix else logits
    ref = LO.sample_from_logits(mixed, kw['use_sampling'], kw['temp'], kw['top_k'], kw['top_p'], noise=noise).squeeze(-1)
    samp = _lib.LMSampling(int(kw['use_sampling']), kw['temp'], kw['top_k'], kw['top_p'], 3.0, 0, 1)
    tok = torch.empty(B, K, dtype=torch.int64, device='cuda')
    ld, nd = logits.cuda(), noise.cuda()
    _lib.check(L.acb_sample(_lib.ptr(ld), _lib.ptr(nd), _lib.ptr(tok), B, rows, K, card, C.byref(samp), 0,
                            _lib.stream()))
    assert torch.equal(tok.cpu(), ref), (tok.cpu() != ref).sum()
    # on-device Philox path: valid ids, reproducible for a (seed, step), different across steps
    samp2 = _lib.LMSampling(1, 1.0, 250, 0.0, 3.0, 1234, 0)
    outs = []
    for step in (0, 0, 1):
        t = torch.empty(B, K, dtype=torch.int64, device='cuda')
        _lib.check(L.acb_sample(_lib.ptr(ld), None, _lib.ptr(t), B, rows, K, card, C.byref(samp2), step, _lib.stream()))
        outs.append(t.cpu())
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], outs[2])
    assert int(outs[0].min()) >= 0 and int(outs[0].max()) < card


def test_philox_sampler_distribution():
    """The on-device sampler draws from the top-k renormalised distribution (chi-square-free check: empirical
    frequencies of a peaked 8-way distribution within 4 sigma over 4000 independent steps)."""
    from audiocraft_b200 import _lib
    import ctypes as C
    L = _lib.lib()
    card = 2048
    logits = torch.full((1, 1, card), -30.0)
    probs = torch.tensor([0.4, 0.2, 0.15, 0.1, 0.06, 0.05, 0.03, 0.01])
    logits[0, 0, :8] = probs.log()
    ld = logits.cuda()
    samp = _lib.LMSampling(1, 1.0, 250, 0.0, 1.0, 99, 0)
    n = 4000
    toks = torch.empty(n, dtype=torch.int64, device='cuda')
    for i in range(n):
        _lib.check(L.acb_sample(_lib.ptr(ld), None, toks[i:i + 1].data_ptr(), 1, 1, 1, card, C.byref(samp), i, _lib.stream()))
    counts = torch.bincount(toks.cpu(), minlength=card)[:8].float()
    sigma = (n * probs * (1 - probs)).sqrt()
    assert ((counts - n * probs).abs() < 4 * sigma + 2).all(), counts


@pytest.mark.parametrize('name', ['lm_mini', 'lm_tiny'])
def test_lm_logits_and_tokens_match(name):
    g = _golden(name)
    cfg, sd, m = _model(name, g['wseed'])
    B, T = g['batch'], g['T']
    _, _, cross = H.lm_condition(cfg, sd, B, g['t_text'], g['cseed'])
    o = LO.LMOracle(sd, cfg, half_gemm=True)
    # teacher-forced along the reference's greedy path
    logits_o = []
    o.generate(None, cross, B, T, use_sampling=False, record_logits=logits_o,
               teacher=LO.build_delay_sequence(g['greedy'], cfg['delays'], cfg['card'])[0])
    seq = o.last_sequence
    lg = m.teacher_forced_logits(seq, cross, cfg['cfg_coef']).cpu()
    ref_half = torch.stack(logits_o)
    err_half = (lg - ref_half).abs().max().item()
    n = g['logits'].shape[0]
    err_ref = (lg[:n] - g['logits']).abs().max().item()
    print(f'{name}: max |logit diff| vs fp16-emulating oracle {err_half:.2e}, vs fp32 reference golden {err_ref:.2e}')
    torch.testing.assert_close(lg, ref_half, rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(lg[:n], g['logits'], rtol=6e-2, atol=6e-2)
    # greedy generation through the public API reproduces the reference tokens
    out = m.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross)
    assert out.shape == g['greedy'].shape and out.dtype == torch.int64
    top2 = ref_half.topk(2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1])
    if not torch.equal(out.cpu(), g['greedy']):
        assert margin.min() < 5e-2, "greedy tokens differ from the reference although every argmax margin is clear"
        pytest.skip(f"greedy path hits an argmax near-tie (min margin {margin.min():.3e}); logits parity holds")
    # sampled generation with injected Exponential(1) noise == oracle with the same noise
    for ki, kw in enumerate((dict(top_k=10, temp=0.9), dict(top_k=0, top_p=0.8), dict(top_k=0, top_p=0.0, temp=1.3))):
        def nf(step, shape, _seed=17 + ki):
            return H.exp_noise(_seed, step, shape[0] * shape[1], shape[2])
        want = o.generate(None, cross, B, T, use_sampling=True, noise_fn=nf, **kw)
        m._debug_noise_fn = lambda step, shape: nf(step, shape).cuda()
        got = m.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=True, cross_attention_src=cross, **kw)
        m._debug_noise_fn = None
        agree = (got.cpu() == want).float().mean().item()
        print(f'{name} sampled {kw}: token agreement {agree:.3f}')
        if agree < 1.0:
            # fp16 logit noise (~1e-2) can flip a draw whose two best p/q scores are nearly tied; everything after the
            # first flip legitimately diverges.  Re-score the first differing step with the oracle along the GPU's own
            # path and require the GPU's pick to be within 3% of the oracle's best score.
            gseq = m.last_sequence.cpu()
            oseq = o.last_sequence
            step = int((gseq != oseq).any(0).any(0).nonzero()[0])
            rec = []
            o.generate(None, cross, B, T, use_sampling=True, noise_fn=nf, record_logits=rec, teacher=gseq, **kw)
            lg = rec[step - 1]
            probs = torch.softmax(lg / kw.get('temp', 1.0), -1)
            if kw.get('top_p', 0.0) > 0:
                ps, pi = LO.top_p_sorted(probs, kw['top_p'])
                score = torch.zeros_like(probs).scatter(-1, pi, ps / nf(step, (B, 4, cfg['card'])).reshape(ps.shape))
            else:
                pf = LO.top_k_filter(probs, kw['top_k']) if kw.get('top_k', 0) > 0 else probs
                score = pf / nf(step, (B, 4, cfg['card'])).reshape(pf.shape)
            valid = LO.delay_sequence_indexes(T, 4, cfg['delays'])[1][:, step]
            picked = score.gather(-1, gseq[..., step].clamp(max=cfg['card'] - 1).unsqueeze(-1)).squeeze(-1)
            rel = (picked / score.max(-1).values)[:, torch.from_numpy(valid)]
            print(f'   first divergence at sequence step {step}: GPU pick / oracle best score = {rel.min():.4f}')
            assert rel.min() > 0.97, "sampled token differs from the oracle although the draw is not a near-tie"
    # prompt continuation keeps the prompt and follows the reference
    prompt = g['greedy'][..., :5].clone()
    got = m.generate(prompt.cuda(), [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross).cpu()
    assert torch.equal(got[..., :5], prompt)
    assert torch.equal(got, g['continuation'])
    got = m.generate(prompt.cuda(), [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross,
                     remove_prompts=True).cpu()
    assert torch.equal(got, g['continuation'][..., 5:])
    # null condition for every row (generate_unconditional)
    got = m.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=False,
                     cross_attention_src=torch.zeros_like(cross)).cpu()
    assert torch.equal(got, g['unconditional'])


def test_musicgen_small_logits_match_reference_golden():
    g = _golden('musicgen_small')
    cfg, sd, m = _model('musicgen_small', g['wseed'])
    _, _, cross = H.lm_condition(cfg, sd, g['batch'], g['t_text'], g['cseed'])
    seq, _ = LO.build_delay_sequence(g['greedy'], cfg['delays'], cfg['card'])
    lg = m.teacher_forced_logits(seq, cross, cfg['cfg_coef']).cpu()
    n = g['logits_top_v'].shape[0]
    got = lg[:n].gather(-1, g['logits_top_i'])
    print('musicgen_small max |logit diff| vs fp32 reference:', (got - g['logits_top_v']).abs().max().item())
    torch.testing.assert_close(got, g['logits_top_v'], rtol=6e-2, atol=6e-2)
    out = m.generate(None, [], num_samples=g['batch'], max_gen_len=g['T'], use_sampling=False, cross_attention_src=cross)
    assert torch.equal(out.cpu(), g['greedy'])


def test_rows_variants_and_batch_independence():
    """rows = 1..34 exercise every row-tile variant of the GEMM; items must not influence each other."""
    cfg, sd, m = _model('lm_tiny', 4)
    for B in (1, 3, 9, 17):
        _, _, cross = H.lm_condition(cfg, sd, B, 4, 2)
        out = m.generate(None, [], num_samples=B, max_gen_len=8, use_sampling=False, cross_attention_src=cross)
        assert out.shape == (B, 4, 8) and int(out.min()) >= 0 and int(out.max()) < cfg['card']
        one = m.generate(None, [], num_samples=1, max_gen_len=8, use_sampling=False,
                         cross_attention_src=torch.cat([cross[B - 1:B], cross[2 * B - 1:]], 0))
        assert torch.equal(one[0], out[B - 1])


def test_musicgen_api_shapes_and_callbacks():
    """Mirror of the reference's tests/models/test_musicgen.py:18-65 on the synthetic small architecture."""
    from audiocraft_b200.loaders import load_compression_model, load_lm_model
    from audiocraft_b200.musicgen import MusicGen
    lm = load_lm_model('synthetic/lm_mini')
    from audiocraft_b200.encodec import EncodecModel
    ccfg = dict(synth.ENCODEC_CONFIGS['encodec_tiny'], bins=lm.card, renormalize=False)   # codec cardinality = LM cardinality
    cm = EncodecModel(synth.synth_encodec_state_dict(ccfg, 1), ccfg)
    cm.set_num_codebooks(4)
    mg = MusicGen('debug', cm, lm, max_duration=30)   # like the reference's debug model (musicgen.py:76-80)
    mg.max_duration = 2.0                              # keep the > max_duration windowing case short
    fr = mg.frame_rate
    assert mg.sample_rate == 16000 and mg.audio_channels == 1
    mg.set_generation_params(duration=1.0, extend_stride=0.5, top_k=40)
    wav, tok = mg.generate_unconditional(2, return_tokens=True)
    assert tok.shape == (2, 4, int(1.0 * fr)) and wav.shape[0] == 2 and wav.shape[1] == 1
    calls = []
    mg.set_custom_progress_callback(lambda a, b: calls.append((a, b)))
    wav, tok = mg.generate(['a tune', 'another one'], progress=True, return_tokens=True)
    assert tok.shape == (2, 4, int(1.0 * fr)) and len(calls) == int(1.0 * fr) + 3 and calls[-1][0] == calls[-1][1]
    x = H.audio_input(cm.cfg, 2, 8000, 1)
    wav, tok = mg.generate_continuation(x, 16000, ['x', None], return_tokens=True)
    assert tok.shape[-1] == int(1.0 * fr)
    # a stereo prompt at another rate goes through convert_audio (resample + downmix) like genmodel.py:183
    x8 = H.audio_input(cm.cfg, 2, 8000 * cm.sample_rate // 16000 // 2, 1)
    wav, tok = mg.generate_continuation(torch.cat([x8, 0.5 * x8], dim=1), cm.sample_rate // 2, ['x', None], return_tokens=True)
    assert tok.shape[-1] == int(1.0 * fr)
    mg.set_generation_params(duration=3.0, extend_stride=1.0)
    wav, tok = mg.generate(['long one'], return_tokens=True)
    assert tok.shape == (1, 4, int(3.0 * fr))
    with pytest.raises(NotImplementedError):
        mg.generate_with_chroma(['x'], None, 16000)


@pytest.mark.parametrize('name,B,T', [('lm_mini', 2, 420), ('lm_medium_2l', 8, 300)])
def test_long_context_attention_matches_oracle(name, B, T):
    """Self attention over long contexts: T teacher-forced steps, so the K / V ring of lm_attn2_kernel (8 warps x 4 positions
    per iteration, 8 iterations deep) wraps many times; the medium case runs at the bench width (rows 16).  CFG-mixed logits
    vs the fp16-emulating oracle."""
    cfg, sd, m = _model(name, 9)
    _, _, cross = H.lm_condition(cfg, sd, B, 5, 4)
    seq = torch.randint(0, cfg['card'], (B, 4, T + 4), generator=torch.Generator().manual_seed(5))
    o = LO.LMOracle(sd, cfg, half_gemm=True)
    rec = []
    o.generate(None, cross, B, T, use_sampling=False, record_logits=rec, teacher=seq)
    ref = torch.stack(rec)
    lg = m.teacher_forced_logits(o.last_sequence, cross, cfg['cfg_coef']).cpu()
    n = ref.shape[0]
    print(f'{name} B={B} T={T}: max |logit diff| vs oracle {(lg[:n] - ref).abs().max():.2e} on |logits| <= {ref.abs().max():.1f}')
    assert torch.isfinite(lg).all()
    torch.testing.assert_close(lg[:n], ref, rtol=2e-2, atol=3e-2)


@pytest.mark.parametrize('name,B', [('lm_medium_2l', 8), ('lm_large_2l', 4), ('lm_medium_2l', 2)])
def test_ft32_tiles_equal_16_feature_tiles(monkeypatch, name, B):
    """The big decode GEMMs (QKV, FFN1, FFN2, heads at d = 1536; FFN2 at d = 2048) use 32-feature tiles by default
    (half the CTAs, half the activation re-reads out of L2); ACB_LM_FT32=0 forces the 16-feature tiles everywhere.  The
    K-split and the per-element summation order are the same, so the logits must be bit-identical."""
    cfg, sd, m = _model(name, 7)
    T = 5
    _, _, cross = H.lm_condition(cfg, sd, B, 6, 2)
    seq = torch.randint(0, cfg['card'], (B, 4, T + 4), generator=torch.Generator().manual_seed(3))
    wide = m.teacher_forced_logits(seq, cross, 3.0).cpu()
    monkeypatch.setenv('ACB_LM_FT32', '0')
    narrow = m.teacher_forced_logits(seq, cross, 3.0).cpu()
    monkeypatch.delenv('ACB_LM_FT32')
    assert torch.isfinite(wide).all()
    assert torch.equal(wide, narrow), f'max diff {(wide - narrow).abs().max():.3e}'


@pytest.mark.parametrize('name,B,ft32', [('lm_medium_2l', 8, '1'), ('lm_medium_2l', 8, '0'), ('lm_large_2l', 4, '1'),
                                         ('lm_large_2l', 32, '1')])
def test_released_widths_match_oracle(monkeypatch, name, B, ft32):
    """MusicGen-medium / -large layer shapes (d = 1536 / 2048, 4d FFN, card 2048) at bench-like row counts
    (rows = 16, 8 and 64 = BASELINE config 5 on one GPU), two layers deep: CFG-mixed logits vs the fp16-emulating oracle."""
    monkeypatch.setenv('ACB_LM_FT32', ft32)   # 32-feature GEMM tiles (default) / 16-feature tiles only
    cfg, sd, m = _model(name, 11)
    _, _, cross = H.lm_condition(cfg, sd, B, 7, 3)
    T = 4
    g = torch.Generator().manual_seed(B)
    seq = torch.randint(0, cfg['card'], (B, 4, T + 4), generator=g)
    o = LO.LMOracle(sd, cfg, half_gemm=True)
    rec = []
    o.generate(None, cross, B, T, use_sampling=False, record_logits=rec, teacher=seq)
    ref = torch.stack(rec)
    # the oracle applies the delay-pattern mask to the teacher (special token where a codebook has no valid step)
    lg = m.teacher_forced_logits(o.last_sequence, cross, cfg['cfg_coef']).cpu()
    print(f'{name} rows={2 * B}: max |logit diff| {(lg - ref).abs().max():.2e} on |logits| <= {ref.abs().max():.1f}')
    torch.testing.assert_close(lg, ref, rtol=2e-2, atol=3e-2)
    out = m.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=True, top_k=250, cross_attention_src=cross)
    assert out.shape == (B, 4, T) and int(out.min()) >= 0 and int(out.max()) < cfg['card']


def test_audiogen_api():
    """AudioGen (SURVEY section 8f.4) rides on the same kernels: 16 kHz codec, 50 Hz frames, its own defaults."""
    from audiocraft_b200.loaders import load_compression_model, load_lm_model
    from audiocraft_b200.musicgen import AudioGen
    from audiocraft_b200.encodec import EncodecModel
    lm = load_lm_model('synthetic/lm_mini')
    ccfg = dict(synth.ENCODEC_CONFIGS['encodec_16k'], bins=lm.card)      # codec cardinality must equal the LM's
    ag = AudioGen('debug', EncodecModel(synth.synth_encodec_state_dict(ccfg, 1), ccfg), lm, max_duration=10)
    assert ag.sample_rate == 16000 and ag.frame_rate == 50 and ag.duration == 5 and ag.extend_stride == 2
    ag.set_generation_params(duration=1.0)
    wav, tok = ag.generate(['dog barking', 'rain'], return_tokens=True)
    assert tok.shape == (2, 4, 50) and wav.shape == (2, 1, 16000)
    assert 'cfg_coef_beta' not in ag.generation_params


@pytest.mark.parametrize('pe', ['rope', 'sin_rope'])
def test_rope_matches_oracle_and_reference_golden(pe):
    """Rotary positions, applied to q and k in the QKV GEMM's epilogue before k is cached (rope.py:84-125 at
    transformer.py:394-395): teacher-forced logits vs the fp16-emulating oracle (2e-2) and the fp32 reference golden (6e-2),
    greedy tokens vs the reference."""
    g = _golden('lm_mini_rope')
    cfg = synth.lm_config('lm_mini')
    cfg['positional_embedding'], cfg['positional_scale'] = pe, g['positional_scale']
    sd = synth.synth_lm_state_dict(cfg, seed=g['wseed'])
    from audiocraft_b200.lm import LMModel
    m = LMModel(sd, cfg, None, None, 'cuda')
    B, T = g['batch'], g['T']
    _, _, cross = H.lm_condition(cfg, sd, B, g['t_text'], g['cseed'])
    seq = H.fullsize_sequence(cfg, B, T, g['sseed'])
    lg = m.teacher_forced_logits(seq, cross, cfg['cfg_coef']).cpu()
    o = LO.LMOracle(sd, cfg, half_gemm=True)
    o.reset()
    outs = [o.forward(torch.cat([seq, seq], 0)[..., t:t + 1], cross) for t in range(seq.shape[-1] - 1)]
    c, u = torch.cat(outs, dim=2).split(B, dim=0)
    want = (u + (c - u) * cfg['cfg_coef']).permute(2, 0, 1, 3)
    print(f'{pe}: max |logit diff| vs oracle {(lg - want).abs().max():.3e}, vs fp32 reference {(lg - g[pe]["logits"]).abs().max():.3e}')
    # observed max 2.2e-2 (rope) and 1.7e-2 (sin_rope) on an H100 (|logits| ~ 20, fp16 weights and fp16 q / k after the
    # rotation): atol 4e-2
    torch.testing.assert_close(lg, want, rtol=2e-2, atol=4e-2)
    torch.testing.assert_close(lg, g[pe]['logits'], rtol=6e-2, atol=6e-2)
    out = m.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross)
    assert torch.equal(out.cpu(), g[pe]['greedy'])


def test_two_step_cfg_matches_reference_golden():
    """two_step_cfg=True (lm.py:376-391): the reference runs the conditional and the null pass separately with their own
    streaming states and mixes with self.cfg_coef (NOT the cfg_coef argument, lm.py:387).  Rows are independent in every
    kernel, so one batched pass is the same arithmetic; the golden tokens come from the reference's literal two-step run."""
    g = _golden('lm_mini_two_step')
    cfg, sd, m = _model('lm_mini', g['wseed'])
    B, T = g['batch'], g['T']
    _, _, cross = H.lm_condition(cfg, sd, B, g['t_text'], g['cseed'])
    out = m.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross,
                     two_step_cfg=True, cfg_coef=1.5).cpu()
    assert torch.equal(out, g['two_step'])
    out = m.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross, cfg_coef=1.5).cpu()
    assert torch.equal(out, g['batched_coef_1p5'])


def test_streaming_state_roundtrip_and_literal_two_step():
    """StreamingModule surface (streaming.py:59-119): get/set_streaming_state restore the decode exactly, the state has
    the reference's keys and shapes ([rows, H, t, 64], offsets [rows]), and a LITERAL two-step CFG -- conditional rows and
    null rows decoded in separate streaming sessions, mixed on the host -- equals the batched pass."""
    cfg, sd, m = _model('lm_mini', 3)
    B, K, card = 2, cfg['n_q'], cfg['card']
    _, _, cross = H.lm_condition(cfg, sd, B, 5, 1)
    gen = torch.Generator().manual_seed(9)
    toks = torch.randint(0, card, (8, B, K), generator=gen)
    m.streaming_begin(B, cross, max_len=16)
    first = [m.streaming_step(toks[i]) for i in range(5)]
    state = m.get_streaming_state()
    assert state['transformer.offsets'].tolist() == [5] * (2 * B)
    assert state['transformer.layers.0.self_attn.past_keys'].shape == (2 * B, cfg['num_heads'], 5, 64)
    a = [m.streaming_step(toks[i]).clone() for i in range(5, 8)]
    m.set_streaming_state(state)
    b = [m.streaming_step(toks[i]).clone() for i in range(5, 8)]
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # literal two-step: cond rows only, then null rows only (coef 1 => the session returns its rows' raw logits)
    m.streaming_begin(B, cross[:B], max_len=16, cfg_coef=1.0)
    lc = [m.streaming_step(toks[i]).clone() for i in range(5)]
    m.streaming_begin(B, cross[B:], max_len=16, cfg_coef=1.0)
    lu = [m.streaming_step(toks[i]).clone() for i in range(5)]
    for i in range(5):
        mixed = lu[i] + (lc[i] - lu[i]) * cfg['cfg_coef']
        torch.testing.assert_close(mixed, first[i], rtol=0, atol=1e-5)
    m.reset_streaming()
    assert int(m._bufs['pos'][0]) == 0


def test_double_cfg_matches_oracle():
    """cfg_coef_beta (MusicGen-Style double CFG, lm.py:362-376) with [cond; style-only; null] rows."""
    cfg, sd, m = _model('lm_mini', 3)
    B, T = 2, 8
    _, _, cross2 = H.lm_condition(cfg, sd, B, 5, 1)
    _, _, other = H.lm_condition(cfg, sd, B, 5, 4)
    cross3 = torch.cat([cross2[:B], other[:B] * 0.5, cross2[B:]], 0)      # a stand-in "style-only" condition in the middle
    o = LO.LMOracle(sd, cfg, half_gemm=True)
    K, special = cfg['n_q'], cfg['card']
    seq = torch.full((B, K, 1), special, dtype=torch.long)
    o.reset()
    want = []
    cur = seq
    m.streaming_begin(B, cross3, max_len=T + 4, cfg_coef=2.0, cfg_coef_beta=3.0)
    for i in range(6):
        tok, lg = o.next_token(cur, cross3, False, 1.0, 0, 0.0, 2.0, None, None, return_logits=True, cfg_coef_beta=3.0)
        got = m.streaming_step(cur[..., 0]).cpu()
        print(f'step {i}: double-CFG logits max diff vs oracle {(got - lg).abs().max():.3e}')
        torch.testing.assert_close(got, lg, rtol=3e-2, atol=3e-2)
        cur = tok
    with pytest.raises(AssertionError):
        m.generate(None, [], num_samples=B, max_gen_len=T, cross_attention_src=cross3)   # 3B rows need cfg_coef_beta


@pytest.mark.parametrize('name,B,T0,pe', [('lm_mini', 2, 9, 'sin'), ('lm_mini', 5, 23, 'sin'), ('lm_medium_2l', 8, 21, 'sin'),
                                           ('lm_mini', 5, 23, 'rope')],
                         ids=['lm_mini-2-9', 'lm_mini-5-23', 'lm_medium_2l-8-21', 'lm_mini-5-23-rope'])
def test_prompt_prefill_equals_token_by_token(monkeypatch, name, B, T0, pe):
    """Prompt prefill (acb_lm_prefill = the reference's multi-token first call, lm.py:513-534, transformer.py:240-247): 64 / rows
    prompt positions per pass through the per-phase kernels on (token, row) pairs, causal inside the pass.  Must leave the same
    KV cache as feeding the prompt one decode step at a time and continue with the same greedy tokens (streaming == batch,
    tests/modules/test_transformer.py:71-85).  The rope case rotates q / k at the position of each (token, row) pair."""
    from audiocraft_b200.lm import LMModel
    cfg = synth.lm_config(name)
    cfg['positional_embedding'] = pe
    sd = synth.synth_lm_state_dict(cfg, seed=5)
    m = LMModel(sd, cfg, None, None)
    T = T0 + 6
    _, _, cross = H.lm_condition(cfg, sd, B, 5, 1)
    prompt = torch.randint(0, cfg['card'], (B, 4, T0), generator=torch.Generator().manual_seed(3))
    out_pf = m.generate(prompt.cuda(), [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross).cpu()
    kc_pf = m._bufs['k_cache'][:, :2 * B, :, :T0].clone()
    vc_pf = m._bufs['v_cache'][:, :2 * B, :, :T0].clone()
    monkeypatch.setenv('ACB_LM_PREFILL', '0')
    out_ss = m.generate(prompt.cuda(), [], num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross).cpu()
    kc_ss = m._bufs['k_cache'][:, :2 * B, :, :T0]
    vc_ss = m._bufs['v_cache'][:, :2 * B, :, :T0]
    print(f'{name} {pe} B={B} T0={T0}: max |K cache diff| {(kc_pf.float() - kc_ss.float()).abs().max():.2e}, '
          f'|V| {(vc_pf.float() - vc_ss.float()).abs().max():.2e}, token agreement {(out_pf == out_ss).float().mean():.4f}')
    torch.testing.assert_close(kc_pf.float(), kc_ss.float(), rtol=0, atol=4e-3)
    torch.testing.assert_close(vc_pf.float(), vc_ss.float(), rtol=0, atol=4e-3)
    assert torch.equal(out_pf[..., :T0], prompt)
    assert (out_pf == out_ss).float().mean() > 0.95
