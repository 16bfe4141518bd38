"""Generate tests/golden/lm_mini_melody.pt by running the REAL reference MusicGen-melody modules on the CPU (found
through oracle/ref_import.py: $AUDIOCRAFT_REFERENCE or baseline/_ref).

    python tests/golden/make_golden_melody.py

The reference LMModel is built with the melody fuser ConditionFuser({'prepend': ['self_wav', 'description'], 'cross': []})
and cross_attention=False (config/conditioner/chroma2music.yaml, lm/default.yaml); `self_wav` is the reference's own
ChromaStemConditioner.  Three things it needs are not installed, and are replaced on the reference side only where the
repository makes the same substitution:
* demucs: the import is stubbed and `_get_stemmed_wav` is replaced by audiocraft_b200.conditioners.identity_stem_separator,
  the stand-in the repository's ChromaStemConditioner is given in the tests;
* librosa.filters.chroma: returns the repository's restated bank (audiocraft_b200.conditioners.chroma_filter_bank), whose
  parity with librosa is unpinned (DESIGN.md section 4); the spectrogram is the reference's torchaudio transform;
* T5: a table of seeded hidden states, as for the other LM goldens.
Weights and inputs are regenerated from seeds (audiocraft_b200/synth.py, tests/helpers.py); only outputs are stored, and
the logits only at a fixed seeded sample of candidate indices to keep the fixture small.
"""
import os
import sys
import types
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import ref_import as R  # noqa: E402
from tests import helpers as H  # noqa: E402
from audiocraft_b200 import synth  # noqa: E402
from audiocraft_b200.conditioners import chroma_filter_bank, identity_stem_separator  # noqa: E402

warnings.filterwarnings('ignore')
torch.set_grad_enabled(False)

NAME = 'lm_mini_melody'
WSEED, CSEED, SSEED, IDX_SEED, N_IDX = 3, 1, 5, 11, 48
PREFIX_STRIDE = 8   # the prefix is stored at every 8th feature: the chroma is stored whole and pins the rest
B, T_TEXT, T = 2, 5, 10
# (case, positional_embedding, match_len_on_eval, melody seconds per item (None = null melody))
CASES = [
    ('sin_melody_null', 'sin', False, (0.5, None)),      # masking by length; a null melody beside a real one
    ('sin_matchlen', 'sin', True, (0.5, 1.5)),           # truncate to chroma_len (the batch is padded to 1.5 s)
    ('sin_matchlen_repeat', 'sin', True, (0.3, 0.3)),    # repeat to chroma_len
    ('sin_null', 'sin', True, (None, None)),             # generate() on a melody model: every melody null
    ('rope_matchlen', 'rope', True, (0.5, 0.3)),
]


def melody_wav(seconds, seed):
    return H.audio_input(dict(sample_rate=32000, channels=1), 1, int(32000 * seconds), seed)


def _stub_demucs():
    demucs = types.ModuleType('demucs')
    pretrained = types.ModuleType('demucs.pretrained')

    class _Sep:
        sources = ['drums', 'bass', 'other', 'vocals']
        samplerate, audio_channels = 44100, 2

        def to(self, *a, **k):
            return self

    pretrained.get_model = lambda name: _Sep()
    demucs.pretrained = pretrained
    sys.modules['demucs'] = demucs
    sys.modules['demucs.pretrained'] = pretrained


def build_ref_melody_lm(cfg, sd, table, pe, match_len):
    R.setup()
    _stub_demucs()
    chroma_mod = R.mod('modules.chroma')
    chroma_mod.filters.chroma = lambda sr, n_fft, tuning, n_chroma: chroma_filter_bank(sr, n_fft, n_chroma).numpy()
    lmm, cond, pat = R.mod('models.lm'), R.mod('modules.conditioners'), R.mod('modules.codebooks_patterns')

    class StubText(cond.TextConditioner):
        def tokenize(self, x):
            hs, ms = zip(*[table['__null__'] if xi is None else table[xi] for xi in x])
            return {'hid': torch.stack(hs), 'mask': torch.stack(ms)}

        def forward(self, inputs):
            mask = inputs['mask']
            return self.output_proj(inputs['hid']) * mask.unsqueeze(-1), mask

    chroma = cond.ChromaStemConditioner(output_dim=cfg['dim'], sample_rate=cfg['sample_rate'], n_chroma=cfg['n_chroma'],
                                        radix2_exp=cfg['radix2_exp'], duration=cfg['duration'],
                                        match_len_on_eval=match_len, device='cpu', argmax=True)
    chroma._get_stemmed_wav = lambda wav, sample_rate: identity_stem_separator(wav, sample_rate)
    prov = cond.ConditioningProvider({'description': StubText(cfg['cond_dim'], cfg['dim']), 'self_wav': chroma},
                                     device='cpu')
    fuser = cond.ConditionFuser({'prepend': ['self_wav', 'description'], 'cross': [], 'sum': [], 'input_interpolate': []})
    kw = dict(n_q=cfg['n_q'], card=cfg['card'], dim=cfg['dim'], num_heads=cfg['num_heads'],
              hidden_scale=cfg['hidden_scale'], norm='layer_norm', norm_first=True, bias_proj=False,
              cfg_coef=cfg['cfg_coef'], num_layers=cfg['num_layers'], bias_ff=False, bias_attn=False, causal=True,
              memory_efficient=pe == 'sin', cross_attention=False, activation='gelu', positional_embedding=pe,
              dropout=0.0)
    if pe != 'sin':   # the streaming rotary offset is right only on the custom attention (see make_golden.golden_lm_rope)
        kw['custom'] = True
    m = lmm.LMModel(pat.DelayedPatternProvider(cfg['n_q'], delays=cfg['delays']), prov, fuser, **kw)
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    assert not unexpected and all(k.endswith(('rope.frequencies', 'spec.window')) for k in missing), (missing, unexpected)
    return m.eval(), cond


def golden_case(pe, match_len, seconds):
    cfg = synth.lm_config(NAME)
    cfg['positional_embedding'] = pe
    sd = synth.synth_lm_state_dict(cfg, seed=WSEED)
    hid, mask, _ = H.lm_condition(cfg, sd, B, T_TEXT, CSEED)
    table = {f'd{i}': (hid[i], mask[i]) for i in range(B)}
    table['__null__'] = (torch.zeros(T_TEXT, cfg['cond_dim']), torch.zeros(T_TEXT, dtype=torch.long))
    m, cond = build_ref_melody_lm(cfg, sd, table, pe, match_len)
    conds = []
    for i, s in enumerate(seconds):
        if s is None:
            wc = cond.WavCondition(torch.zeros(1, 1, 1), torch.tensor([0]), sample_rate=[32000], path=[None])
        else:
            w = melody_wav(s, 100 + i)
            wc = cond.WavCondition(w, torch.tensor([w.shape[-1]]), sample_rate=[32000], path=[None])
        conds.append(cond.ConditioningAttributes(text={'description': f'd{i}'}, wav={'self_wav': wc}))
    null = cond.ClassifierFreeGuidanceDropout(p=1.0)(conds)
    tokenized = m.condition_provider.tokenize(conds + null)
    chroma = m.condition_provider.conditioners['self_wav']._get_wav_embedding(tokenized['self_wav'])
    ct = m.condition_provider(tokenized)
    prefix, _ = m.fuser(torch.zeros(2 * B, 0, cfg['dim']), ct)
    seq = H.fullsize_sequence(cfg, B, T, SSEED)
    lg = m(torch.cat([seq, seq], 0)[..., :-1], conditions=[], condition_tensors=ct)   # [2B, K, S-1, card]
    c, u = lg.split(B, dim=0)
    mixed = (u + (c - u) * cfg['cfg_coef']).permute(2, 0, 1, 3).contiguous()             # [S-1, B, K, card]
    idx = torch.randperm(cfg['card'], generator=torch.Generator().manual_seed(IDX_SEED))[:N_IDX].sort().values
    greedy = m.generate(None, conds, max_gen_len=T, use_sampling=False)
    return dict(pe=pe, match_len_on_eval=match_len, seconds=seconds, chroma=chroma.clone(),
                self_wav_mask=ct['self_wav'][1].clone(), prefix_len=prefix.shape[1],
                prefix_stride=PREFIX_STRIDE, prefix_strided=prefix[..., ::PREFIX_STRIDE].clone(),
                logits_idx=idx, logits=mixed[..., idx].clone(), greedy=greedy)


if __name__ == '__main__':
    out = dict(name=NAME, batch=B, t_text=T_TEXT, T=T, wseed=WSEED, cseed=CSEED, sseed=SSEED, melody_seed0=100,
               cases={})
    for case, pe, ml, secs in CASES:
        out['cases'][case] = golden_case(pe, ml, secs)
        g = out['cases'][case]
        print(case, 'prefix', g['prefix_len'], 'greedy', tuple(g['greedy'].shape))
    torch.save(out, os.path.join(H.GOLDEN_DIR, f'{NAME}.pt'))
