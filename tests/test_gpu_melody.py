"""GPU tests of MusicGen-melody: the condition prefix prefilled into the KV cache (acb_lm_begin_prefix) and the decode step
running at cache position P + t, through LMModel and MusicGen.generate_with_chroma.
Tolerances are the LM policy of tests/test_gpu_lm.py: K/V caches of two prefill orders atol 4e-3; logits vs the
fp16-emulating oracle atol/rtol 2e-2, vs the fp32 oracle atol 6e-2; greedy tokens agree except at near-ties."""
import pytest
import torch

from tests import helpers as H
from tests import melody_golden as MG
from tests.prefix_oracle import PrefixLMOracle
from audiocraft_b200 import synth

pytestmark = pytest.mark.gpu


def _model(name, pe='sin', seed=5):
    from audiocraft_b200.lm import LMModel
    cfg = synth.lm_config(name)
    cfg['positional_embedding'] = pe
    sd = synth.synth_lm_state_dict(cfg, seed=seed)
    return cfg, sd, LMModel(sd, cfg, None, None)


def _prefix(cfg, rows, P, seed):
    """[rows, P, d] condition prefix: distinct cond and null rows, magnitudes like output_proj outputs."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(rows, P, cfg['dim'], generator=g) * 0.5


def _cross(cfg, sd, B):
    return H.lm_condition(cfg, sd, B, 5, 1)[2] if cfg['cross_attention'] else None


@pytest.mark.parametrize('name,B,P,T0,pe', [
    ('lm_mini', 3, 37, 7, 'sin'),            # rows 6: 10 positions per pass, P not a multiple
    ('lm_mini_melody', 5, 23, 0, 'rope'),    # no cross attention, rotary positions
    ('lm_medium_2l', 8, 251, 5, 'sin'),      # rows 16 (the benchmark batch): 4 positions per pass, 251 = 62 * 4 + 3
])
def test_prefix_prefill_equals_one_position_per_pass(monkeypatch, name, B, P, T0, pe):
    """The prefix passes (64 / rows positions each, causal inside a pass) leave the KV cache that one position per pass
    leaves, and the prompt prefill and greedy decode that follow at cache position P + t agree."""
    cfg, sd, m = _model(name, pe)
    T = T0 + 6
    rows = 2 * B
    prefix = _prefix(cfg, rows, P, 11)
    cross = _cross(cfg, sd, B)
    prompt = torch.randint(0, cfg['card'], (B, 4, T0), generator=torch.Generator().manual_seed(3)) if T0 else None
    kw = dict(num_samples=B, max_gen_len=T, use_sampling=False, cross_attention_src=cross, prefix=prefix)
    out_pf = m.generate(None if prompt is None else prompt.cuda(), [], **kw).cpu()
    n = P + T0
    kc_pf = m._bufs['k_cache'][:, :rows, :, :n].clone()
    vc_pf = m._bufs['v_cache'][:, :rows, :, :n].clone()
    monkeypatch.setenv('ACB_LM_PREFILL_PER', '1')
    out_1 = m.generate(None if prompt is None else prompt.cuda(), [], **kw).cpu()
    kc_1 = m._bufs['k_cache'][:, :rows, :, :n]
    vc_1 = m._bufs['v_cache'][:, :rows, :, :n]
    print(f'{name} {pe} B={B} P={P} T0={T0}: max |K diff| {(kc_pf.float() - kc_1.float()).abs().max():.2e}, '
          f'|V| {(vc_pf.float() - vc_1.float()).abs().max():.2e}, token agreement {(out_pf == out_1).float().mean():.4f}')
    torch.testing.assert_close(kc_pf.float(), kc_1.float(), rtol=0, atol=4e-3)
    torch.testing.assert_close(vc_pf.float(), vc_1.float(), rtol=0, atol=4e-3)
    if prompt is not None:
        assert torch.equal(out_pf[..., :T0], prompt)
    assert (out_pf == out_1).float().mean() > 0.95


@pytest.mark.parametrize('name,B,P,pe', [('lm_mini_melody', 2, 29, 'sin'), ('lm_mini', 3, 12, 'sin'),
                                         ('lm_mini_melody', 2, 17, 'sin_rope')])
def test_prefix_logits_match_oracle(name, B, P, pe):
    """Teacher-forced CFG logits with a prefix (with and without cross attention) vs the fp16-emulating oracle (2e-2) and
    the fp32 oracle (6e-2)."""
    cfg, sd, m = _model(name, pe)
    S = 24
    seq = H.fullsize_sequence(cfg, B, S - max(cfg['delays']) - 1, 4)
    prefix = _prefix(cfg, 2 * B, P, 13)
    cross = _cross(cfg, sd, B)
    out = m.teacher_forced_logits(seq, cross, cfg['cfg_coef'], prefix=prefix).cpu()
    for half, tol in ((True, 2e-2), (False, 6e-2)):
        ref = PrefixLMOracle(sd, cfg, half_gemm=half, prefix=prefix).teacher_forced_mixed(seq, cross, cfg['cfg_coef'])
        err = (out - ref).abs().max().item()
        print(f'{name} {pe} P={P} half={half}: max |logit diff| {err:.3e}')
        torch.testing.assert_close(out, ref, atol=tol, rtol=tol)


def _melody_model():
    from audiocraft_b200.loaders import load_musicgen
    mg = load_musicgen('synthetic/lm_mini_melody')
    mg.set_generation_params(use_sampling=False, duration=0.5)
    return mg


def _melody(B, seconds, seed):
    cfg = dict(sample_rate=32000, channels=1)
    return H.audio_input(cfg, B, int(32000 * seconds), seed)


def _assert_greedy(got, want, oracle_logits, what):
    """The project's greedy rule: tokens equal, or a skip when the fp16-emulating oracle's own argmax margin along the path
    shows a near-tie (tests/test_gpu_lm.py)."""
    got = got.cpu()
    if torch.equal(got, want):
        return
    top2 = torch.stack(oracle_logits).topk(2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1]).min().item()
    assert margin < 5e-2, f"{what}: greedy tokens differ although every argmax margin is clear (min {margin:.3e})"
    pytest.skip(f"{what}: greedy path hits an argmax near-tie (min margin {margin:.3e})")


def _oracle_greedy(sd, cfg, prefix, B, T, prompt=None):
    rec = []
    o = PrefixLMOracle(sd, cfg, half_gemm=True, prefix=prefix)
    out = o.generate(prompt, None, B, T, use_sampling=False, cfg_coef=cfg['cfg_coef'], record_logits=rec)
    return out, rec


def _golden_lm(case):
    from audiocraft_b200.lm import LMModel
    g = MG.golden()
    cfg = MG.config(g, case)
    sd = MG.weights(g, cfg)
    prov, fuser = MG.provider_and_fuser(g, case, cfg, sd)
    return g, cfg, sd, LMModel(sd, cfg, prov, fuser, 'cuda')


@pytest.mark.parametrize('case', ['sin_melody_null', 'sin_matchlen', 'sin_matchlen_repeat', 'sin_null', 'rope_matchlen'])
def test_melody_lm_matches_reference_golden(case):
    """The reference's MusicGen-melody LM (tests/golden/make_golden_melody.py) against the device: teacher-forced CFG logits
    with the [chroma ; description] prefix within 6e-2 of the reference's fp32 ones (and 2e-2 of the fp16-emulating
    oracle), and LMModel.generate from the conditions (chroma front-end included) gives the reference's greedy tokens."""
    g, cfg, sd, m = _golden_lm(case)
    c = g['cases'][case]
    B, T = g['batch'], g['T']
    _, _, prefix = MG.repo_conditions(g, case, cfg, sd)
    seq = MG.teacher_sequence(g, cfg)
    lg = m.teacher_forced_logits(seq, None, cfg['cfg_coef'], prefix=prefix).cpu()
    half = PrefixLMOracle(sd, cfg, half_gemm=True, prefix=prefix).teacher_forced_mixed(seq, None, cfg['cfg_coef'])
    err_ref = (lg[..., c['logits_idx']] - c['logits']).abs().max().item()
    print(f'{case}: max |logit diff| vs reference golden {err_ref:.3e}, vs fp16-emulating oracle '
          f'{(lg - half).abs().max().item():.3e}')
    torch.testing.assert_close(lg[..., c['logits_idx']], c['logits'], rtol=6e-2, atol=6e-2)
    torch.testing.assert_close(lg, half, rtol=2e-2, atol=2e-2)
    out = m.generate(None, MG.attributes(g, case, 'cuda'), max_gen_len=T, use_sampling=False)
    _, rec = _oracle_greedy(sd, cfg, prefix, B, T)
    _assert_greedy(out, c['greedy'], rec, case)


def _golden_musicgen(case):
    from audiocraft_b200.loaders import load_compression_model
    from audiocraft_b200.musicgen import MusicGen
    g, cfg, sd, lm = _golden_lm(case)
    mg = MusicGen('golden/lm_mini_melody', load_compression_model('synthetic/encodec_32k', 'cuda', 1), lm, max_duration=30)
    mg.set_generation_params(use_sampling=False, duration=g['T'] / mg.frame_rate)
    return g, cfg, sd, mg


def test_generate_with_chroma_matches_reference_golden():
    """MusicGen.generate_with_chroma end to end (melody -> chroma, matched to the training length -> prefix -> LM -> codec)
    gives the reference's greedy tokens; generate() on the melody model (every melody null) gives the reference's
    null-melody tokens."""
    case = 'sin_matchlen'
    g, cfg, sd, mg = _golden_musicgen(case)
    wav, tokens = mg.generate_with_chroma(['d0', 'd1'], MG.melodies(g, case), 32000, return_tokens=True)
    assert tokens.shape == (g['batch'], 4, g['T']) and wav.shape[0] == g['batch']
    _, _, prefix = MG.repo_conditions(g, case, cfg, sd)
    _, rec = _oracle_greedy(sd, cfg, prefix, g['batch'], g['T'])
    _assert_greedy(tokens, g['cases'][case]['greedy'], rec, 'generate_with_chroma')
    _, t_gen = mg.generate(['d0', 'd1'], return_tokens=True)
    _, prefix0 = mg.lm._condition_tensors(MG.attributes(g, 'sin_null', 'cuda'))
    _, rec0 = _oracle_greedy(sd, cfg, prefix0, g['batch'], g['T'])
    _assert_greedy(t_gen, g['cases']['sin_null']['greedy'], rec0, 'generate (null melody)')


def test_generate_unconditional_on_melody_model_uses_null_chroma():
    """generate_unconditional on a melody model carries a null `self_wav` (musicgen.py:212-217) and null descriptions:
    its tokens are generate_with_chroma's with [None] descriptions and melodies."""
    mg = _melody_model()
    _, t_unc = mg.generate_unconditional(2, return_tokens=True)
    _, t_none = mg.generate_with_chroma([None, None], [None, None], 32000, return_tokens=True)
    assert torch.equal(t_unc, t_none)


def test_generate_continuation_on_melody_model():
    """A prefix, then the prompt prefill, then decode: the prompt's tokens come back first and the continuation equals
    the fp16-emulating oracle fed the same prefix and prompt (or hits a near-tie)."""
    mg = _melody_model()
    prompt_wav = _melody(2, 0.2, 9)
    _, tokens = mg.generate_continuation(prompt_wav, 32000, ['jazz', None], return_tokens=True)
    attributes, prompt_tokens = mg._prepare_tokens_and_attributes(['jazz', None], prompt_wav.cuda())
    assert torch.equal(tokens[..., :prompt_tokens.shape[-1]], prompt_tokens)
    _, prefix = mg.lm._condition_tensors(attributes)
    sd = synth.synth_lm_state_dict(mg.lm.cfg_dict, seed=0, device='cuda', dtype=torch.float16)   # as load_lm_model draws them
    want, rec = _oracle_greedy(sd, mg.lm.cfg_dict, prefix, 2, tokens.shape[-1], prompt_tokens.cpu())
    _assert_greedy(tokens, want, rec, 'continuation')


def test_long_generation_slices_the_melody_per_window(monkeypatch):
    """Beyond max_duration every window is conditioned on max_duration seconds of the melody from the window's start,
    wrapped around periodically (musicgen.py:308-323); a null melody stays null."""
    mg = _melody_model()
    mg.max_duration = 0.6
    mg.set_generation_params(use_sampling=False, duration=1.3, extend_stride=0.3)
    melody = _melody(1, 0.45, 5)
    seen = []
    orig = mg.lm.generate

    def spy(prompt, attributes, **kw):
        seen.append([a.wav['self_wav'] for a in attributes])
        return orig(prompt, attributes, **kw)
    monkeypatch.setattr(mg.lm, 'generate', spy)
    _, tokens = mg.generate_with_chroma(['x', 'y'], [melody[0], None], 32000, return_tokens=True)
    assert tokens.shape[-1] == int(1.3 * mg.frame_rate)
    assert len(seen) >= 3
    L, target = melody.shape[-1], int(0.6 * 32000)
    for w, conds in enumerate(seen):
        start = int(w * int(0.3 * mg.frame_rate) / mg.frame_rate * 32000)   # the window's start, in whole frames
        want = melody[0][..., (torch.arange(start, start + target)) % L]
        torch.testing.assert_close(conds[0].wav.cpu()[0], want, rtol=0, atol=0)
        assert int(conds[0].length.item()) == target
        assert conds[1].wav.shape[-1] == 1 and int(conds[1].length.item()) == 0


def test_prefix_refusals():
    mg = _melody_model()
    attributes, _ = mg._prepare_tokens_and_attributes(['a'], None)
    with pytest.raises(NotImplementedError):
        mg.lm.generate(None, attributes, max_gen_len=8, two_step_cfg=True)
    with pytest.raises(NotImplementedError):
        mg.lm.generate(None, attributes, max_gen_len=8, cfg_coef_beta=2.0)


def test_streaming_state_includes_prefix():
    """streaming_begin prefills the prefix; offsets and past_keys count it, as the reference's transformer offsets do.
    Streaming steps give the teacher-forced logits, and so do steps after a state is saved, the stream reset (the prefix
    stays cached: the reference prepends it again after a reset) and the state restored."""
    cfg, sd, m = _model('lm_mini_melody')
    B, P = 2, 9
    prefix = _prefix(cfg, 2 * B, P, 3)
    seq = H.fullsize_sequence(cfg, B, 8, 2)
    want = m.teacher_forced_logits(seq, None, cfg['cfg_coef'], prefix=prefix, n_steps=6).cpu()
    m.streaming_begin(B, None, 16, prefix=prefix)
    st = m.get_streaming_state()
    assert int(st['transformer.offsets'][0]) == P
    assert st['transformer.layers.0.self_attn.past_keys'].shape[2] == P
    got = torch.stack([m.streaming_step(seq[..., i].cuda()).cpu() for i in range(3)])
    torch.testing.assert_close(got, want[:3], rtol=0, atol=0)
    saved = m.get_streaming_state()
    assert int(saved['transformer.offsets'][0]) == P + 3
    assert saved['transformer.layers.0.self_attn.past_keys'].shape[2] == P + 3
    # reset: back to the state right after the prefix; the first step again gives step 0's logits
    m.reset_streaming()
    assert int(m.get_streaming_state()['transformer.offsets'][0]) == P
    torch.testing.assert_close(m.streaming_step(seq[..., 0].cuda()).cpu(), want[0], rtol=0, atol=0)
    # restore the saved state (3 tokens after the prefix) and continue
    m.set_streaming_state(saved)
    got = torch.stack([m.streaming_step(seq[..., i].cuda()).cpu() for i in range(3, 6)])
    torch.testing.assert_close(got, want[3:6], rtol=0, atol=0)
    assert int(m.get_streaming_state()['transformer.offsets'][0]) == P + 6
