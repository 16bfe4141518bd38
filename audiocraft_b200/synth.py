"""Architecture tables and seeded synthetic weights in the REFERENCE state_dict layout.

There are no pretrained checkpoints (and no network) in the build or GPU image, so tests, smoke()
and bench.py use random-init weights of the named architectures.  Keys and shapes follow the
reference checkpoints (SURVEY.md section 8b; audiocraft/models/loaders.py:78-126 consumes
``best_state`` dicts with exactly this layout), so the same dict loads into the reference modules,
the CPU oracle and the CUDA models.

Hyper-parameters restate the reference config tree (read-only source of shapes):
  config/model/encodec/default.yaml + encodec_large_nq4_s640.yaml / encodec_base_causal.yaml,
  config/model/lm/musicgen_lm.yaml + model_scale/{small,medium,large}.yaml.
"""
import math
import typing as tp

import torch

# ----------------------------------------------------------------------------- EnCodec

ENCODEC_CONFIGS: tp.Dict[str, dict] = {
    # MusicGen's codec: 32 kHz mono, hop 640 (50 Hz), 4 x 2048 codes, non-causal.
    'encodec_32k': dict(channels=1, dimension=128, n_filters=64, n_residual_layers=1, ratios=[8, 5, 4, 4],
                        kernel_size=7, last_kernel_size=7, residual_kernel_size=3, dilation_base=2,
                        causal=False, pad_mode='reflect', compress=2, lstm=2, norm='weight_norm',
                        trim_right_ratio=1.0, sample_rate=32000, n_q=4, bins=2048, renormalize=False,
                        latent_sigma=0.35),
    # AudioGen's codec (config/model/encodec/encodec_large_nq4_s320.yaml): 16 kHz, hop 320 (50 Hz), 4 x 2048 codes.
    'encodec_16k': dict(channels=1, dimension=128, n_filters=64, n_residual_layers=1, ratios=[8, 5, 4, 2],
                        kernel_size=7, last_kernel_size=7, residual_kernel_size=3, dilation_base=2,
                        causal=False, pad_mode='reflect', compress=2, lstm=2, norm='weight_norm',
                        trim_right_ratio=1.0, sample_rate=16000, n_q=4, bins=2048, renormalize=False,
                        latent_sigma=0.35),
    # AudioCraft base 24 kHz causal codec (BASELINE config 1), hop 320 (75 Hz).
    'encodec_24k': dict(channels=1, dimension=128, n_filters=32, n_residual_layers=1, ratios=[8, 5, 4, 2],
                        kernel_size=7, last_kernel_size=7, residual_kernel_size=3, dilation_base=2,
                        causal=True, pad_mode='reflect', compress=2, lstm=2, norm='weight_norm',
                        trim_right_ratio=1.0, sample_rate=24000, n_q=8, bins=1024, renormalize=False,
                        latent_sigma=0.35),
    # Small shapes for fast parity tests (same code paths: odd stride, dilation, 2 residual layers).
    'encodec_tiny': dict(channels=1, dimension=32, n_filters=8, n_residual_layers=2, ratios=[5, 4, 2],
                         kernel_size=7, last_kernel_size=7, residual_kernel_size=3, dilation_base=2,
                         causal=False, pad_mode='reflect', compress=2, lstm=2, norm='weight_norm',
                         trim_right_ratio=1.0, sample_rate=16000, n_q=4, bins=64, renormalize=True,
                         latent_sigma=0.35),
    'encodec_tiny_causal': dict(channels=2, dimension=32, n_filters=8, n_residual_layers=1, ratios=[4, 3],
                                kernel_size=7, last_kernel_size=7, residual_kernel_size=3, dilation_base=2,
                                causal=True, pad_mode='reflect', compress=2, lstm=1, norm='weight_norm',
                                trim_right_ratio=1.0, sample_rate=16000, n_q=3, bins=48, renormalize=False,
                                latent_sigma=0.35),
}

# GroupNorm codecs (norm='time_group_norm'): their state dicts hold each conv's GroupNorm next to it (`...conv.norm.*`,
# `...convtr.norm.*`), outside the conv prefixes of the layer plan.
ENCODEC_GN_CONFIGS: tp.Dict[str, dict] = {
    # facebook/encodec_48khz (transformers EncodecConfig of that repo): 48 kHz stereo, hop 320 (150 Hz), 16 x 1024 codes,
    # GroupNorm(1, C) after every convolution, 1x1 conv shortcuts; transformers cuts its input into 1 s chunks
    'encodec_48k': dict(channels=2, dimension=128, n_filters=32, n_residual_layers=1, ratios=[8, 5, 4, 2],
                        kernel_size=7, last_kernel_size=7, residual_kernel_size=3, dilation_base=2,
                        causal=False, pad_mode='reflect', compress=2, lstm=2, norm='time_group_norm', true_skip=False,
                        trim_right_ratio=1.0, sample_rate=48000, n_q=16, bins=1024, renormalize=True,
                        latent_sigma=0.35),
}


def encodec_hop(cfg: dict) -> int:
    return int(math.prod(cfg['ratios']))


def encodec_frame_rate(cfg: dict) -> float:
    return cfg['sample_rate'] / encodec_hop(cfg)


def encodec_layers(cfg: dict) -> tp.Dict[str, tp.List[dict]]:
    """Ordered layer plan of the SEANet encoder and decoder with the reference module indices
    (audiocraft/modules/seanet.py:113-150, 207-254).  Each entry:
      kind 'conv'  : prefix, cin, cout, k, stride, dilation, elu (ELU before), res ('in' saves the skip,
                     'out' adds it, 'shortcut' = the 1x1 conv that produces the skip when true_skip is off)
      kind 'convtr': prefix, cin, cout, k, stride, elu
      kind 'lstm'  : prefix, dim, layers
    """
    nf, dim, ch = cfg['n_filters'], cfg['dimension'], cfg['channels']
    rk, ks, lks = cfg['residual_kernel_size'], cfg['kernel_size'], cfg['last_kernel_size']

    def res_entries(prefix, c, j):
        hid = c // cfg['compress']
        out = []
        if not cfg.get('true_skip', True):   # SEANetResnetBlock with a 1x1 conv shortcut (seanet.py:54-57)
            out.append(dict(kind='conv', prefix=f'{prefix}shortcut.conv.conv.', cin=c, cout=c, k=1, stride=1,
                            dilation=1, elu=False, res='shortcut'))
        out += [dict(kind='conv', prefix=f'{prefix}block.1.conv.conv.', cin=c, cout=hid, k=rk, stride=1,
                     dilation=cfg['dilation_base'] ** j, elu=True, res='in'),
                dict(kind='conv', prefix=f'{prefix}block.3.conv.conv.', cin=hid, cout=c, k=1, stride=1,
                     dilation=1, elu=True, res='out')]
        return out

    enc: tp.List[dict] = []
    i, mult = 0, 1
    enc.append(dict(kind='conv', prefix=f'encoder.model.{i}.conv.conv.', cin=ch, cout=nf, k=ks, stride=1,
                    dilation=1, elu=False, res=None))
    i += 1
    for ratio in reversed(cfg['ratios']):
        for j in range(cfg['n_residual_layers']):
            enc += res_entries(f'encoder.model.{i}.', mult * nf, j)
            i += 1
        i += 1
        enc.append(dict(kind='conv', prefix=f'encoder.model.{i}.conv.conv.', cin=mult * nf, cout=mult * nf * 2,
                        k=2 * ratio, stride=ratio, dilation=1, elu=True, res=None))
        i += 1
        mult *= 2
    if cfg['lstm']:
        enc.append(dict(kind='lstm', prefix=f'encoder.model.{i}.lstm.', dim=mult * nf, layers=cfg['lstm']))
        i += 1
    i += 1
    enc.append(dict(kind='conv', prefix=f'encoder.model.{i}.conv.conv.', cin=mult * nf, cout=dim, k=lks, stride=1,
                    dilation=1, elu=True, res=None))

    dec: tp.List[dict] = []
    i, mult = 0, 2 ** len(cfg['ratios'])
    dec.append(dict(kind='conv', prefix=f'decoder.model.{i}.conv.conv.', cin=dim, cout=mult * nf, k=ks, stride=1,
                    dilation=1, elu=False, res=None))
    i += 1
    if cfg['lstm']:
        dec.append(dict(kind='lstm', prefix=f'decoder.model.{i}.lstm.', dim=mult * nf, layers=cfg['lstm']))
        i += 1
    for ratio in cfg['ratios']:
        i += 1
        dec.append(dict(kind='convtr', prefix=f'decoder.model.{i}.convtr.convtr.', cin=mult * nf,
                        cout=mult * nf // 2, k=2 * ratio, stride=ratio, elu=True))
        i += 1
        for j in range(cfg['n_residual_layers']):
            dec += res_entries(f'decoder.model.{i}.', mult * nf // 2, j)
            i += 1
        mult //= 2
    i += 1
    dec.append(dict(kind='conv', prefix=f'decoder.model.{i}.conv.conv.', cin=nf, cout=ch, k=lks, stride=1,
                    dilation=1, elu=True, res=None))
    return {'encoder': enc, 'decoder': dec}


def _uniform(gen, shape, bound, device, dtype=torch.float32):
    return ((torch.rand(shape, generator=gen, device=device, dtype=torch.float32) * 2 - 1) * bound).to(dtype)


def synth_encodec_state_dict(cfg: dict, seed: int = 0, device='cpu') -> tp.Dict[str, torch.Tensor]:
    """Seeded random EnCodec weights (variance-preserving conv init, weight-norm g perturbed so that the
    fold g*v/|v| is exercised, codebooks scaled to the latent statistics).  norm='time_group_norm' adds each conv's GroupNorm
    gamma / beta (`...conv.norm.*`, `...convtr.norm.*`) drawn around 1 / 0, so a transposed gamma or a dropped beta shows."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    sd: tp.Dict[str, torch.Tensor] = {}
    plan = encodec_layers(cfg)
    for layer in plan['encoder'] + plan['decoder']:
        p = layer['prefix']
        if layer['kind'] == 'lstm':
            hdim = layer['dim']
            b = 1.0 / math.sqrt(hdim)
            for n in range(layer['layers']):
                sd[f'{p}weight_ih_l{n}'] = _uniform(gen, (4 * hdim, hdim), b, device)
                sd[f'{p}weight_hh_l{n}'] = _uniform(gen, (4 * hdim, hdim), b, device)
                sd[f'{p}bias_ih_l{n}'] = _uniform(gen, (4 * hdim,), b, device)
                sd[f'{p}bias_hh_l{n}'] = _uniform(gen, (4 * hdim,), b, device)
            continue
        cin, cout, k = layer['cin'], layer['cout'], layer['k']
        if layer['kind'] == 'conv':
            shape, fan_in = (cout, cin, k), cin * k
        else:  # ConvTranspose1d weight is [Cin, Cout, K]; each output sees 2 taps per input channel (K = 2*stride)
            shape, fan_in = (cin, cout, k), cin * k // layer['stride']
        v = _uniform(gen, shape, math.sqrt(3.0 / fan_in), device)
        if cfg['norm'] == 'weight_norm':
            nrm = v.reshape(shape[0], -1).norm(dim=1).reshape(-1, 1, 1)
            g = nrm * (1.0 + 0.1 * torch.randn(nrm.shape, generator=gen, device=device))
            sd[p + 'weight_g'] = g
            sd[p + 'weight_v'] = v
        else:
            sd[p + 'weight'] = v
        sd[p + 'bias'] = _uniform(gen, (cout,), 0.05, device)
        if cfg['norm'] == 'time_group_norm':
            n = p.rsplit('.', 2)[0] + '.norm.'
            sd[n + 'weight'] = 1.0 + 0.2 * torch.randn((cout,), generator=gen, device=device)
            sd[n + 'bias'] = 0.1 * torch.randn((cout,), generator=gen, device=device)
    sigma = cfg.get('latent_sigma', 1.0)
    for q in range(cfg['n_q']):
        emb = torch.randn((cfg['bins'], cfg['dimension']), generator=gen, device=device) * (sigma * 0.6 ** q)
        p = f'quantizer.vq.layers.{q}._codebook.'
        sd[p + 'embed'] = emb
        sd[p + 'embed_avg'] = emb.clone()
        sd[p + 'cluster_size'] = torch.ones(cfg['bins'], device=device)
        sd[p + 'inited'] = torch.ones(1, device=device)
    return sd


# ----------------------------------------------------------------------------- LM

# stereo MusicGen (docs/MUSICGEN.md "Training stereo models", config/solver/musicgen/default.yaml:20-29): the codec's 4
# codebooks of the left and of the right channel interleaved as `b (k c) t`, both channels of a level on the same delay
_STEREO = dict(n_q=8, delays=[0, 0, 1, 1, 2, 2, 3, 3])
_MELODY = dict(cross_attention=False, cond_dim=768, n_chroma=12, radix2_exp=14, duration=30.0, sample_rate=32000)

LM_CONFIGS: tp.Dict[str, dict] = {
    'musicgen_small': dict(dim=1024, num_heads=16, num_layers=24),
    'musicgen_medium': dict(dim=1536, num_heads=24, num_layers=48),
    'musicgen_large': dict(dim=2048, num_heads=32, num_layers=48),
    'lm_tiny': dict(dim=128, num_heads=2, num_layers=2, card=64),
    'lm_mini': dict(dim=256, num_heads=4, num_layers=3, card=128, cond_dim=96),
    # the released widths with only 2 layers: exercise the d = 1536 / 2048 GEMM tiling in tests without the full depth
    'lm_medium_2l': dict(dim=1536, num_heads=24, num_layers=2, card=2048, cond_dim=64),
    'lm_large_2l': dict(dim=2048, num_heads=32, num_layers=2, card=2048, cond_dim=64),
    # MusicGen-melody (config/conditioner/chroma2music.yaml): no cross attention, the prefix [chroma ; T5-base description]
    # is prepended; 12 chroma bins from a 2^14-sample STFT at 32 kHz, 30 s training segments
    'musicgen_melody': dict(dim=1536, num_heads=24, num_layers=48, cross_attention=False, cond_dim=768, n_chroma=12,
                            radix2_exp=14, duration=30.0, sample_rate=32000),
    'lm_mini_melody': dict(dim=256, num_heads=4, num_layers=3, card=2048, cond_dim=96, cross_attention=False, n_chroma=12,
                           radix2_exp=14, duration=1.0, sample_rate=32000),
    'musicgen_stereo_small': dict(dim=1024, num_heads=16, num_layers=24, **_STEREO),
    'musicgen_stereo_medium': dict(dim=1536, num_heads=24, num_layers=48, **_STEREO),
    'musicgen_stereo_large': dict(dim=2048, num_heads=32, num_layers=48, **_STEREO),
    'musicgen_stereo_melody': dict(dim=1536, num_heads=24, num_layers=48, **_MELODY, **_STEREO),
    'musicgen_stereo_melody_large': dict(dim=2048, num_heads=32, num_layers=48, **_MELODY, **_STEREO),
    # stereo test shapes: card 2048 keeps the released heads width n_q * card = 16384
    'lm_mini_stereo': dict(dim=256, num_heads=4, num_layers=3, card=2048, cond_dim=96, **_STEREO),
    'lm_medium_2l_stereo': dict(dim=1536, num_heads=24, num_layers=2, card=2048, cond_dim=64, **_STEREO),
    'lm_mini_melody_stereo': dict(dim=256, num_heads=4, num_layers=3, card=2048, cond_dim=96, cross_attention=False,
                                  n_chroma=12, radix2_exp=14, duration=1.0, sample_rate=32000, **_STEREO),
}
_LM_COMMON = dict(hidden_scale=4, n_q=4, card=2048, delays=[0, 1, 2, 3], max_period=10000.0,
                  positional_scale=1.0, cross_attention=True, cfg_coef=3.0, cond_dim=768)


def lm_config(name: str) -> dict:
    cfg = dict(_LM_COMMON)
    cfg.update(LM_CONFIGS[name])
    cfg['name'] = name
    return cfg


def synth_lm_state_dict(cfg: dict, seed: int = 0, device='cpu', dtype=torch.float32) -> tp.Dict[str, torch.Tensor]:
    """Seeded random LM weights, gaussian std 1/sqrt(fan_in) scaled by 1/sqrt(2*depth) per layer like the
    reference's 'gaussian' + depthwise 'current' init (audiocraft/models/lm.py:40-72, 176-208)."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    d, L, K, card = cfg['dim'], cfg['num_layers'], cfg['n_q'], cfg['card']
    ff = int(cfg['hidden_scale'] * d)

    def gauss(shape, fan_in, depth=None):
        std = 1.0 / math.sqrt(fan_in)
        if depth is not None:
            std /= math.sqrt(2 * depth)
        # generate in chunks of rows to bound peak memory for the 3.3B model
        out = torch.empty(shape, device=device, dtype=dtype)
        rows = shape[0]
        step = max(1, (1 << 24) // max(1, shape[1]))
        for r in range(0, rows, step):
            n = min(step, rows - r)
            out[r:r + n] = (torch.randn((n, shape[1]), generator=gen, device=device) * std).to(dtype)
        return out

    sd: tp.Dict[str, torch.Tensor] = {}
    for k in range(K):
        sd[f'emb.{k}.weight'] = gauss((card + 1, d), d)
    for li in range(L):
        p = f'transformer.layers.{li}.'
        depth = li + 1
        sd[p + 'self_attn.in_proj_weight'] = gauss((3 * d, d), d, depth)
        sd[p + 'self_attn.out_proj.weight'] = gauss((d, d), d, depth)
        if cfg['cross_attention']:
            sd[p + 'cross_attention.in_proj_weight'] = gauss((3 * d, d), d, depth)
            sd[p + 'cross_attention.out_proj.weight'] = gauss((d, d), d, depth)
            sd[p + 'norm_cross.weight'] = (1.0 + 0.1 * torch.randn(d, generator=gen, device=device)).float()
            sd[p + 'norm_cross.bias'] = (0.05 * torch.randn(d, generator=gen, device=device)).float()
        sd[p + 'linear1.weight'] = gauss((ff, d), d, depth)
        sd[p + 'linear2.weight'] = gauss((d, ff), ff, depth)
        for n in ('norm1', 'norm2'):
            sd[p + n + '.weight'] = (1.0 + 0.1 * torch.randn(d, generator=gen, device=device)).float()
            sd[p + n + '.bias'] = (0.05 * torch.randn(d, generator=gen, device=device)).float()
    sd['out_norm.weight'] = (1.0 + 0.1 * torch.randn(d, generator=gen, device=device)).float()
    sd['out_norm.bias'] = (0.05 * torch.randn(d, generator=gen, device=device)).float()
    for k in range(K):
        sd[f'linears.{k}.weight'] = gauss((card, d), d) * 4.0  # a peaked-enough next-token distribution
    cd = cfg['cond_dim']
    sd['condition_provider.conditioners.description.output_proj.weight'] = gauss((d, cd), cd)
    sd['condition_provider.conditioners.description.output_proj.bias'] = \
        (0.05 * torch.randn(d, generator=gen, device=device)).to(dtype)
    if cfg.get('n_chroma'):   # drawn last: the text-only configurations keep their weights
        nc = cfg['n_chroma']
        sd['condition_provider.conditioners.self_wav.output_proj.weight'] = gauss((d, nc), nc)
        sd['condition_provider.conditioners.self_wav.output_proj.bias'] = \
            (0.05 * torch.randn(d, generator=gen, device=device)).to(dtype)
    return sd


def synth_text_condition(cfg: dict, batch: int, t_text: int, seed: int = 0, device='cpu'):
    """Stand-in for the T5 encoder output (outside the hot path, SURVEY.md section 8f.3): seeded
    [B, T_text, cond_dim] hidden states and an attention mask with ragged lengths."""
    gen = torch.Generator(device='cpu')
    gen.manual_seed(seed + 7919)
    hid = torch.randn((batch, t_text, cfg['cond_dim']), generator=gen)
    lengths = torch.randint(max(1, t_text // 2), t_text + 1, (batch,), generator=gen)
    mask = (torch.arange(t_text).view(1, -1) < lengths.view(-1, 1)).long()
    return hid.to(device), mask.to(device)


# ----------------------------------------------------------------------------- T5 text encoder

# transformers' T5Config of the released checkpoints the conditioners name (config/conditioner/text2music.yaml: t5-base,
# text2sound.yaml: t5-large)
T5_CONFIGS: tp.Dict[str, dict] = {
    't5-small': dict(d_model=512, d_kv=64, d_ff=2048, num_heads=8, num_layers=6),
    't5-base': dict(d_model=768, d_kv=64, d_ff=3072, num_heads=12, num_layers=12),
    't5-large': dict(d_model=1024, d_kv=64, d_ff=4096, num_heads=16, num_layers=24),
}


def t5_config(name: str) -> dict:
    """The config.json fields of a released T5 (relu feed-forward, 32128-token vocabulary, 32 buckets up to distance 128)."""
    cfg = dict(model_type='t5', vocab_size=32128, relative_attention_num_buckets=32, relative_attention_max_distance=128,
               layer_norm_epsilon=1e-6, feed_forward_proj='relu', dropout_rate=0.1, initializer_factor=1.0,
               is_encoder_decoder=True, pad_token_id=0, eos_token_id=1, decoder_start_token_id=0)
    cfg.update(T5_CONFIGS[name])
    cfg['num_decoder_layers'] = cfg['num_layers']
    return cfg


def synth_t5_state_dict(cfg: dict, seed: int = 0, wi_scale: float = 1.0) -> tp.Dict[str, torch.Tensor]:
    """Seeded fp32 T5 encoder weights in transformers' key layout, drawn with transformers' T5 init scales (q: (d d_kv)^-1/2;
    k, v, o, wi, relative bias: d^-1/2; wo: d_ff^-1/2; embedding 1; norms 1).  Unscaled N(0, 1) weights would be meaningless
    without T5's attention scale, which the init folds into q.  wi_scale multiplies every wi (tests of large activations)."""
    gen = torch.Generator()
    gen.manual_seed(seed)
    d, dkv, ff, H, L = cfg['d_model'], cfg['d_kv'], cfg['d_ff'], cfg['num_heads'], cfg['num_layers']

    def normal(shape, std):
        return torch.randn(shape, generator=gen) * std

    sd = {'shared.weight': normal((cfg['vocab_size'], d), 1.0)}
    for i in range(L):
        a, f = f'encoder.block.{i}.layer.0.', f'encoder.block.{i}.layer.1.'
        sd[a + 'SelfAttention.q.weight'] = normal((H * dkv, d), (d * dkv) ** -0.5)
        sd[a + 'SelfAttention.k.weight'] = normal((H * dkv, d), d ** -0.5)
        sd[a + 'SelfAttention.v.weight'] = normal((H * dkv, d), d ** -0.5)
        sd[a + 'SelfAttention.o.weight'] = normal((d, H * dkv), (H * dkv) ** -0.5)
        if i == 0:
            sd[a + 'SelfAttention.relative_attention_bias.weight'] = normal((cfg['relative_attention_num_buckets'], H), d ** -0.5)
        sd[a + 'layer_norm.weight'] = torch.ones(d)
        sd[f + 'DenseReluDense.wi.weight'] = normal((ff, d), d ** -0.5) * wi_scale
        sd[f + 'DenseReluDense.wo.weight'] = normal((d, ff), ff ** -0.5)
        sd[f + 'layer_norm.weight'] = torch.ones(d)
    sd['encoder.final_layer_norm.weight'] = torch.ones(d)
    return sd


def write_t5_dir(path: str, cfg: dict, state_dict: tp.Dict[str, torch.Tensor], spiece_model: str, fmt: str = 'safetensors'):
    """A local T5 directory in Hugging Face layout: config.json, model.safetensors (fmt 'safetensors') or pytorch_model.bin
    (fmt 'bin'), and a copy of the SentencePiece model `spiece_model` as spiece.model."""
    import json
    import os
    import shutil
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, 'config.json'), 'w') as fh:
        json.dump(cfg, fh, indent=1)
    sd = {k: v.contiguous() for k, v in state_dict.items()}
    if fmt == 'safetensors':
        from safetensors.torch import save_file
        save_file(sd, os.path.join(path, 'model.safetensors'))
    elif fmt == 'bin':
        torch.save(sd, os.path.join(path, 'pytorch_model.bin'))
    else:
        raise ValueError(f"fmt {fmt!r}: 'safetensors' or 'bin'")
    shutil.copyfile(spiece_model, os.path.join(path, 'spiece.model'))
    return path
