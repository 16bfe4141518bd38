"""The repository side of tests/golden/lm_mini_melody.pt (written by tests/golden/make_golden_melody.py from the reference's
MusicGen-melody modules): the same seeded weights, text hidden states and melodies, fed through this package's conditioners."""
import os

import torch

from tests import helpers as H
from audiocraft_b200 import conditioners as CD
from audiocraft_b200 import synth

NAME = 'lm_mini_melody'


def golden():
    return torch.load(os.path.join(H.GOLDEN_DIR, f'{NAME}.pt'), weights_only=False)


def config(g, case):
    cfg = synth.lm_config(NAME)
    cfg['positional_embedding'] = g['cases'][case]['pe']
    return cfg


def weights(g, cfg):
    return synth.synth_lm_state_dict(cfg, seed=g['wseed'])


def text_encoder(g, cfg, sd):
    """PrecomputedTextConditioner encoder: 'd<i>' -> the golden's seeded hidden states of item i, '' -> zeros."""
    hid, mask, _ = H.lm_condition(cfg, sd, g['batch'], g['t_text'], g['cseed'])

    def encode(entries):
        hs = [hid[int(e[1:])] if e else torch.zeros_like(hid[0]) for e in entries]
        ms = [mask[int(e[1:])] if e else torch.zeros_like(mask[0]) for e in entries]
        return torch.stack(hs), torch.stack(ms)
    return encode


def melodies(g, case):
    """Per item: the [1, T] melody at 32 kHz, or None for a null melody."""
    out = []
    for i, s in enumerate(g['cases'][case]['seconds']):
        out.append(None if s is None else H.audio_input(dict(sample_rate=32000, channels=1), 1, int(32000 * s),
                                                          g['melody_seed0'] + i)[0])
    return out


def provider_and_fuser(g, case, cfg, sd, device='cpu'):
    """This package's description + chroma conditioners with the golden's weights, and the melody fuser."""
    c = g['cases'][case]
    text = CD.PrecomputedTextConditioner(cfg['cond_dim'], cfg['dim'], text_encoder(g, cfg, sd))
    chroma = CD.ChromaStemConditioner(cfg['dim'], cfg['sample_rate'], cfg['n_chroma'], cfg['radix2_exp'], cfg['duration'],
                                      match_len_on_eval=c['match_len_on_eval'], argmax=True,
                                      stem_separator=CD.identity_stem_separator)
    prov = CD.ConditioningProvider({'description': text, 'self_wav': chroma})
    cp = {k[len('condition_provider.'):]: v.float() for k, v in sd.items() if k.startswith('condition_provider.')}
    prov.load_state_dict(cp, strict=False)
    return prov.to(device), CD.ConditionFuser({'prepend': ['self_wav', 'description'], 'cross': []})


def attributes(g, case, device='cpu'):
    """ConditioningAttributes of the case, as MusicGen._prepare_tokens_and_attributes builds them."""
    out = []
    for i, mel in enumerate(melodies(g, case)):
        if mel is None:
            wc = CD.WavCondition(torch.zeros((1, 1, 1), device=device), torch.tensor([0], device=device), [32000], [None])
        else:
            wc = CD.WavCondition(mel[None].to(device), torch.tensor([mel.shape[-1]], device=device), [32000], [None])
        out.append(CD.ConditioningAttributes(text={'description': f'd{i}'}, wav={'self_wav': wc}))
    return out


@torch.no_grad()
def repo_conditions(g, case, cfg, sd):
    """(chroma, self_wav mask, prefix) of [conditions ; null conditions] computed by this package on the CPU."""
    prov, fuser = provider_and_fuser(g, case, cfg, sd)
    tok = prov.tokenize(attributes(g, case) + CD.nullify_all(attributes(g, case)))
    chroma = prov.conditioners['self_wav']._get_wav_embedding(tok['self_wav'])
    tensors = prov(tok)
    return chroma, tensors['self_wav'][1], fuser.prefix_source(tensors)


def teacher_sequence(g, cfg):
    return H.fullsize_sequence(cfg, g['batch'], g['T'], g['sseed'])
