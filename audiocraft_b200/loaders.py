"""Model assembly (mirror of the parts of audiocraft/models/loaders.py + builders.py the path needs).

The reference resolves names through the HF hub and re-instantiates modules from an omegaconf ``xp.cfg``
(loaders.py:78-126, builders.py:70-175).  Here: a checkpoint in the reference's export format
(``{'best_state': state_dict, 'xp.cfg': yaml}``, utils/export.py:20-79) found on local disk is loaded with the
hyper-parameters read from its yaml (PyYAML; omegaconf is not in the image), and ``synthetic/<arch>`` builds seeded
random weights of a released architecture (no pretrained weights exist offline).
"""
import os
import typing as tp

import torch

from . import synth
from .conditioners import (ChromaStemConditioner, ConditionFuser, ConditioningProvider, PrecomputedTextConditioner,
                           T5Conditioner, identity_stem_separator)
from .encodec import EncodecModel
from .lm import LMModel

_SCALES = {'small': 'musicgen_small', 'medium': 'musicgen_medium', 'large': 'musicgen_large', 'melody': 'musicgen_melody',
           'stereo-small': 'musicgen_stereo_small', 'stereo-medium': 'musicgen_stereo_medium',
           'stereo-large': 'musicgen_stereo_large', 'stereo-melody': 'musicgen_stereo_melody',
           'stereo-melody-large': 'musicgen_stereo_melody_large'}
# the released stereo checkpoints' xp.cfg (config/solver/musicgen/default.yaml:20-29): the codec's codebooks of both channels
# interleaved as `b (k c) t`, 4 codebooks per channel
_STEREO_WRAP = dict(interleave_stereo_codebooks={'use': True, 'per_timestep': False}, compression_model_n_q=4)


def _cfg_from_yaml(text: str) -> dict:
    import yaml
    return yaml.safe_load(text)


def _load_pkg(path: str) -> dict:
    """Exported checkpoints hold tensors, a yaml STRING and version strings (utils/export.py:20-79), so they load with
    weights_only=True; unpickling arbitrary objects from a user-supplied path needs the explicit opt-in
    AUDIOCRAFT_B200_UNSAFE_LOAD=1."""
    try:
        return torch.load(path, map_location='cpu', weights_only=True)
    except Exception:
        if os.environ.get('AUDIOCRAFT_B200_UNSAFE_LOAD') == '1':
            return torch.load(path, map_location='cpu', weights_only=False)
        raise


_T5_DIMS = {'t5-small': 512, 't5-base': 768, 't5-large': 1024, 't5-3b': 1024, 't5-11b': 1024,
            'google/flan-t5-small': 512, 'google/flan-t5-base': 768, 'google/flan-t5-large': 1024,
            'google/flan-t5-xl': 2048, 'google/flan-t5-xxl': 4096}   # conditioners.py:436-448


def lm_cfg_from_xp(xp: dict) -> dict:
    """Hyper-parameters of an exported LM checkpoint from its xp.cfg (what builders.get_lm_model reads,
    builders.py:136-175), restricted to what the decode kernels implement; anything else raises instead of silently
    computing a different model."""
    tl = xp['transformer_lm']
    unsupported = []
    if not tl.get('norm_first', False):
        unsupported.append('norm_first=false (post-norm)')
    for b in ('bias_proj', 'bias_ff', 'bias_attn'):
        if tl.get(b, False):
            unsupported.append(f'{b}=true')
    if tl.get('layer_scale', None) is not None:
        unsupported.append('layer_scale')
    if tl.get('norm', 'layer_norm') != 'layer_norm':
        unsupported.append(f"norm={tl.get('norm')}")
    if tl.get('activation', 'gelu') != 'gelu':
        unsupported.append(f"activation={tl.get('activation')}")
    if tl.get('qk_layer_norm', False) or tl.get('qk_layer_norm_cross', False):
        unsupported.append('qk_layer_norm')
    if tl.get('kv_repeat', 1) != 1:
        unsupported.append('kv_repeat')
    if tl.get('past_context', None) is not None:
        unsupported.append('past_context')
    pe = tl.get('positional_embedding', 'sin')
    if pe not in ('sin', 'rope', 'sin_rope') or tl.get('xpos', False):
        unsupported.append(f'positional_embedding={pe} xpos={tl.get("xpos", False)}')
    if xp.get('codebooks_pattern', {}).get('modeling', 'delay') != 'delay':
        unsupported.append(f"codebooks_pattern.modeling={xp['codebooks_pattern'].get('modeling')}")
    fz = xp.get('fuser', {})
    for how in ('sum', 'input_interpolate'):
        if fz.get(how):
            unsupported.append(f'fuser.{how}={fz[how]}')
    prepend = list(fz.get('prepend') or [])
    if prepend and (prepend not in (['self_wav', 'description'], ['self_wav'])):
        unsupported.append(f'fuser.prepend={prepend} (only the melody layouts [self_wav, description] / [self_wav])')
    if list(fz.get('cross', [])) not in (['description'], []):
        unsupported.append(f"fuser.cross={fz.get('cross')}")
    if fz.get('cross_attention_pos_emb', False):
        unsupported.append('fuser.cross_attention_pos_emb')
    isc = xp.get('interleave_stereo_codebooks') or {}
    if isc.get('use') and isc.get('per_timestep'):
        unsupported.append('interleave_stereo_codebooks.per_timestep=true (codes interleaved along time)')
    if unsupported:
        raise NotImplementedError("this checkpoint's LM is outside what the decode kernels implement: " + ', '.join(unsupported))
    chroma = None
    if 'self_wav' in prepend:
        sw = xp.get('conditioners', {}).get('self_wav') or {}
        if sw.get('model') != 'chroma_stem':
            raise NotImplementedError(f"self_wav conditioner '{sw.get('model')}' is not built (only chroma_stem)")
        cs = sw['chroma_stem']
        if cs.get('eval_wavs') is not None:
            raise NotImplementedError("chroma_stem.eval_wavs (evaluation wavs from a dataset) is not built")
        if cs.get('cache_path') is not None:
            raise NotImplementedError("chroma_stem.cache_path (the chroma embedding cache) is not built")
        chroma = dict(n_chroma=int(cs['n_chroma']), radix2_exp=int(cs['radix2_exp']), argmax=bool(cs.get('argmax', True)),
                      match_len_on_eval=bool(cs.get('match_len_on_eval', True)),
                      sample_rate=int(cs.get('sample_rate') or xp['sample_rate']),
                      duration=float(xp['dataset']['segment_duration']))   # builders.py: duration = segment_duration
    cond_dim, t5 = None, None
    desc = xp.get('conditioners', {}).get('description')
    if desc is not None:
        if desc.get('model') != 't5':
            raise NotImplementedError(f"description conditioner '{desc.get('model')}' is not built (only t5)")
        t5 = dict(desc['t5'])
        cond_dim = _T5_DIMS.get(t5['name'])
        if cond_dim is None:
            raise NotImplementedError(f"unknown T5 variant {t5['name']}")
    return dict(dim=tl['dim'], num_heads=tl['num_heads'], num_layers=tl['num_layers'], hidden_scale=tl.get('hidden_scale', 4),
                n_q=tl['n_q'], card=tl['card'], delays=list(xp['codebooks_pattern']['delay']['delays']),
                max_period=float(tl.get('max_period', 10000.0)), positional_scale=float(tl.get('positional_scale', 1.0)),
                positional_embedding=pe, cross_attention=bool(fz.get('cross')),
                cfg_coef=xp['classifier_free_guidance']['inference_coef'], cond_dim=cond_dim,
                two_step_cfg=tl.get('two_step_cfg', False), prepend=prepend, chroma=chroma, t5=t5)


def _text_conditioner(cfg: dict, text_encoder, device):
    """The description conditioner: a T5Conditioner when `text_encoder` is a local T5 directory, else the caller's callable
    returning (hidden states, mask) behind a PrecomputedTextConditioner."""
    if isinstance(text_encoder, (str, os.PathLike)):
        from .t5 import read_config
        path = os.fspath(text_encoder)
        if not os.path.isdir(path):
            raise FileNotFoundError(f"text_encoder '{path}' is not a local T5 directory (names are not resolved on a hub)")
        d_model = read_config(path)['d_model']
        if d_model != cfg['cond_dim']:
            name = (cfg.get('t5') or {}).get('name', 'the checkpoint\'s T5')
            raise ValueError(f"T5 directory {path} has d_model {d_model}, but {name} has {cfg['cond_dim']}")
        t5 = cfg.get('t5') or {}
        return T5Conditioner(path, cfg['dim'], finetune=bool(t5.get('finetune', False)), device=device,
                             word_dropout=float(t5.get('word_dropout', 0.)), normalize_text=bool(t5.get('normalize_text', False)))
    return PrecomputedTextConditioner(cfg['cond_dim'], cfg['dim'], text_encoder)


def _melody_parts(cfg: dict, text_encoder, stem_separator, device):
    """Provider and fuser of a prepend (melody) model: description (when prepended) + chroma_stem self_wav."""
    ch = cfg['chroma']
    conds = {}
    if 'description' in cfg['prepend']:
        conds['description'] = _text_conditioner(cfg, text_encoder, device)
    conds['self_wav'] = ChromaStemConditioner(cfg['dim'], ch['sample_rate'], ch['n_chroma'], ch['radix2_exp'], ch['duration'],
                                              match_len_on_eval=ch['match_len_on_eval'], argmax=ch['argmax'],
                                              stem_separator=stem_separator)
    return ConditioningProvider(conds), ConditionFuser({'prepend': list(cfg['prepend']), 'cross': []})


def load_compression_model(name: str, device='cuda', seed: int = 0) -> EncodecModel:
    if name.startswith('synthetic/'):
        arch = name.split('/', 1)[1]
        cfg = synth.ENCODEC_CONFIGS.get(arch) or synth.ENCODEC_GN_CONFIGS[arch]
        return EncodecModel(synth.synth_encodec_state_dict(cfg, seed), cfg, device)
    if os.path.isfile(name):
        pkg = _load_pkg(name)
        if 'pretrained' in pkg:
            raise RuntimeError(f"{name} redirects to '{pkg['pretrained']}' (HF hub); no network in this image")
        xp = _cfg_from_yaml(pkg['xp.cfg']) if isinstance(pkg['xp.cfg'], str) else pkg['xp.cfg']
        sea, rvq = xp['seanet'], xp['rvq']
        cfg = dict(channels=xp['channels'], dimension=sea['dimension'], n_filters=sea['n_filters'],
                   n_residual_layers=sea['n_residual_layers'], ratios=list(sea['ratios']),
                   kernel_size=sea['kernel_size'], last_kernel_size=sea['last_kernel_size'],
                   residual_kernel_size=sea['residual_kernel_size'], dilation_base=sea['dilation_base'],
                   causal=xp['encodec']['causal'], pad_mode=sea['pad_mode'], compress=sea['compress'],
                   lstm=sea['lstm'], norm=sea['norm'], norm_params=dict(sea.get('norm_params') or {}),
                   trim_right_ratio=(sea.get('decoder') or {}).get('trim_right_ratio', 1.0),   # seanet.decoder.* (encodec/default.yaml)
                   sample_rate=xp['sample_rate'], n_q=rvq['n_q'], bins=rvq['bins'],
                   renormalize=xp['encodec']['renormalize'])
        return EncodecModel(pkg['best_state'], cfg, device)
    raise FileNotFoundError(f"compression model '{name}': not a local checkpoint and not 'synthetic/<arch>' "
                            "(the HF hub is unreachable from this image)")


def synthetic_text_encoder(cfg: dict, t_text: int = 16, seed: int = 0):
    """Deterministic stand-in for the frozen T5 encoder (weights unavailable offline): hidden states are a seeded
    function of the prompt string, lengths follow the word count."""
    def encode(entries: tp.List[str]):
        hs, ms = [], []
        for e in entries:
            g = torch.Generator()
            g.manual_seed((hash_str(e) + seed) % (2 ** 31))
            hs.append(torch.randn((t_text, cfg['cond_dim']), generator=g))
            n = max(1, min(t_text, len(e.split()) + 1))
            ms.append((torch.arange(t_text) < n).long())
        return torch.stack(hs), torch.stack(ms)
    return encode


def hash_str(s: str) -> int:
    h = 2166136261
    for ch in s.encode():
        h = ((h ^ ch) * 16777619) & 0xffffffff
    return h


def load_lm_model(name: str, device='cuda', seed: int = 0, text_encoder=None, stem_separator=None) -> LMModel:
    """`stem_separator`: callable (wav [B,C,T], sample_rate) -> melody stems [B,1,T] standing in for Demucs in a melody
    checkpoint; `synthetic/melody` uses `identity_stem_separator` (the mono mix is the melody) when none is given."""
    if name.startswith('synthetic/'):
        arch = name.split('/', 1)[1]
        cfg = synth.lm_config(_SCALES.get(arch, arch))
        sd = synth.synth_lm_state_dict(cfg, seed, device=device, dtype=torch.float16)
        enc = text_encoder or synthetic_text_encoder(cfg)
        if cfg.get('n_chroma'):
            cfg = dict(cfg, prepend=['self_wav', 'description'],
                       chroma=dict(n_chroma=cfg['n_chroma'], radix2_exp=cfg['radix2_exp'], argmax=True, match_len_on_eval=False,
                                   sample_rate=cfg['sample_rate'], duration=cfg['duration']))
            provider, fuser = _melody_parts(cfg, enc, stem_separator or identity_stem_separator, device)
            return LMModel(sd, cfg, provider, fuser, device)
        provider = ConditioningProvider({'description': _text_conditioner(cfg, enc, device)})
        return LMModel(sd, cfg, provider, ConditionFuser({'cross': ['description']}), device)
    if os.path.isfile(name):
        pkg = _load_pkg(name)
        xp = _cfg_from_yaml(pkg['xp.cfg']) if isinstance(pkg['xp.cfg'], str) else pkg['xp.cfg']
        cfg = lm_cfg_from_xp(xp)
        provider = None
        if cfg['prepend']:
            if stem_separator is None:
                raise RuntimeError("this checkpoint is melody-conditioned: pass stem_separator=<callable (wav [B,C,T], "
                                   "sample_rate) -> melody stems [B,1,T]> standing in for Demucs (htdemucs weights are not "
                                   "available offline)")
            if 'description' in cfg['prepend'] and text_encoder is None:
                raise RuntimeError("this checkpoint is text-conditioned: pass text_encoder=<local T5 directory> or <callable "
                                   f"returning the frozen T5 hidden states [B,T,{cfg['cond_dim']}] and attention mask>")
            provider, fuser = _melody_parts(cfg, text_encoder, stem_separator, device)
            return LMModel(pkg['best_state'], cfg, provider, fuser, device)
        if cfg['cross_attention']:
            if text_encoder is None:
                raise RuntimeError("this checkpoint is text-conditioned: pass text_encoder=<local T5 directory in Hugging Face "
                                   "layout> or <callable returning the frozen T5 hidden states "
                                   f"[B,T,{cfg['cond_dim']}] and attention mask>")
            provider = ConditioningProvider({'description': _text_conditioner(cfg, text_encoder, device)})
        return LMModel(pkg['best_state'], cfg, provider, ConditionFuser({'cross': ['description']}), device)
    raise FileNotFoundError(f"LM '{name}': not a local checkpoint and not 'synthetic/<scale>'")


def _wrap_from_xp(cm, lm_ckpt: str):
    """builders.get_wrapped_compression_model (builders.py:338-351): the LM checkpoint's xp.cfg says whether its codebooks
    are interleaved stereo and how many codebooks of the codec it models."""
    from .encodec import get_wrapped_compression_model
    pkg = _load_pkg(lm_ckpt)
    xp = _cfg_from_yaml(pkg['xp.cfg']) if isinstance(pkg['xp.cfg'], str) else pkg['xp.cfg']
    return get_wrapped_compression_model(cm, xp.get('interleave_stereo_codebooks'), xp.get('compression_model_n_q'))


def load_musicgen(name: str, device=None, seed: int = 0, text_encoder=None, stem_separator=None):
    """`text_encoder`: a local T5 directory in Hugging Face layout (config.json, model.safetensors or pytorch_model.bin,
    spiece.model), run on the device by T5Conditioner, or a callable list[str] -> (hidden [B,T,cond_dim], mask [B,T]) giving
    the frozen T5's output (the reference instantiates T5 from the HF hub, conditioners.py:422-515).
    `stem_separator`: the Demucs stand-in a melody checkpoint needs (see load_lm_model)."""
    from .musicgen import MusicGen
    device = 'cuda' if device is None else device
    if name.startswith('synthetic/'):
        lm = load_lm_model(name, device, seed, text_encoder, stem_separator)
        cm = load_compression_model('synthetic/encodec_32k', device, seed + 1)
        if name.split('/', 1)[1].startswith('stereo-'):
            from .encodec import get_wrapped_compression_model
            cm = get_wrapped_compression_model(cm, **_STEREO_WRAP)
        return MusicGen(name, cm, lm, max_duration=30)
    if os.path.isdir(name):
        lm_path = os.path.join(name, 'state_dict.bin')
        lm = load_lm_model(lm_path, device, text_encoder=text_encoder, stem_separator=stem_separator)
        cm = _wrap_from_xp(load_compression_model(os.path.join(name, 'compression_state_dict.bin'), device), lm_path)
        return MusicGen(name, cm, lm, max_duration=30)
    raise FileNotFoundError(f"MusicGen '{name}': pass a local checkpoint directory or 'synthetic/<scale>' "
                            f"({', '.join(_SCALES)})")


def load_audiogen(name: str, device=None, seed: int = 0, text_encoder=None):
    """`synthetic/audiogen-medium` (seeded random weights of the released architecture) or a local checkpoint directory;
    `text_encoder` as for load_musicgen."""
    from .musicgen import AudioGen
    device = 'cuda' if device is None else device
    if name.startswith('synthetic/'):
        scale = name.split('/', 1)[1].replace('audiogen-', '')
        lm = load_lm_model(f'synthetic/{scale}', device, seed, text_encoder)
        cm = load_compression_model('synthetic/encodec_16k', device, seed + 1)
        return AudioGen(name, cm, lm, max_duration=10)
    if os.path.isdir(name):
        lm_path = os.path.join(name, 'state_dict.bin')
        lm = load_lm_model(lm_path, device, text_encoder=text_encoder)
        cm = _wrap_from_xp(load_compression_model(os.path.join(name, 'compression_state_dict.bin'), device), lm_path)
        return AudioGen(name, cm, lm, max_duration=10)
    raise FileNotFoundError(f"AudioGen '{name}': pass a local checkpoint directory or 'synthetic/audiogen-medium'")
