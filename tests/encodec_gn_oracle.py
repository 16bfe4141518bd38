"""CPU oracle of the GroupNorm EnCodec (norm='time_group_norm') and of the chunked encode / decode with linear overlap-add that
transformers runs for the 48 kHz codec.  Plain fp32 torch ops on the reference-layout state dict, built on the primitives of
oracle/encodec_oracle.py; every function restates the algorithm and cites where it lives.

GroupNorm placement (audiocraft/modules/conv.py:91-137): NormConv1d / NormConvTranspose1d run conv -> GroupNorm(1, C), and
StreamableConvTranspose1d trims AFTER that (conv.py:221-243), so a transposed conv's statistics include the trimmed steps.
"""
import torch
import torch.nn.functional as F

from oracle import encodec_oracle as EO


def group_norm(y, sd, prefix, eps=1e-5):
    """nn.GroupNorm(1, C) of `prefix` (weight / bias), or y unchanged when the layer has none (norm='none' blocks)."""
    if prefix + 'weight' not in sd:
        return y
    return F.group_norm(y, 1, sd[prefix + 'weight'].float(), sd[prefix + 'bias'].float(), eps)


def conv(x, sd, prefix, cfg, stride=1, dilation=1):
    """StreamableConv1d: `prefix` = '<...>.conv.' holding conv.* and norm.*."""
    w, b = EO._conv_weight(sd, prefix + 'conv.')
    y = EO.sconv1d(x, w, b, stride=stride, dilation=dilation, causal=cfg['causal'], pad_mode=cfg['pad_mode'])
    return group_norm(y, sd, prefix + 'norm.')


def convtr(x, sd, prefix, cfg, stride):
    """StreamableConvTranspose1d (non-causal): full transposed conv, GroupNorm, then the fixed trim."""
    w, b = EO._conv_weight(sd, prefix + 'convtr.')
    y = group_norm(F.conv_transpose1d(x, w, b, stride=stride), sd, prefix + 'norm.')
    total = w.shape[-1] - stride
    right = total // 2
    return y[..., total - right: y.shape[-1] - right]


def resblock(x, sd, prefix, cfg, dilation):
    """SEANetResnetBlock.forward, audiocraft/modules/seanet.py:36-60: shortcut(x) + block(x)."""
    y = conv(EO.elu(x), sd, prefix + 'block.1.conv.', cfg, dilation=dilation)
    y = conv(EO.elu(y), sd, prefix + 'block.3.conv.', cfg)
    skip = x if cfg.get('true_skip', True) else conv(x, sd, prefix + 'shortcut.conv.', cfg)
    return skip + y


def encode_latent(x, sd, cfg):
    """SEANetEncoder.forward, module indices as built at audiocraft/modules/seanet.py:113-150."""
    i = 0
    x = conv(x, sd, f'encoder.model.{i}.conv.', cfg)
    i += 1
    for ratio in reversed(cfg['ratios']):
        for j in range(cfg['n_residual_layers']):
            x = resblock(x, sd, f'encoder.model.{i}.', cfg, cfg['dilation_base'] ** j)
            i += 1
        i += 1
        x = conv(EO.elu(x), sd, f'encoder.model.{i}.conv.', cfg, stride=ratio)
        i += 1
    if cfg['lstm']:
        x = EO.lstm_block(x, sd, f'encoder.model.{i}.lstm.', cfg['lstm'])
        i += 1
    i += 1
    return conv(EO.elu(x), sd, f'encoder.model.{i}.conv.', cfg)


def decode_latent(z, sd, cfg):
    """SEANetDecoder.forward, module indices as built at audiocraft/modules/seanet.py:207-254."""
    i = 0
    x = conv(z, sd, f'decoder.model.{i}.conv.', cfg)
    i += 1
    if cfg['lstm']:
        x = EO.lstm_block(x, sd, f'decoder.model.{i}.lstm.', cfg['lstm'])
        i += 1
    for ratio in cfg['ratios']:
        i += 1
        x = convtr(EO.elu(x), sd, f'decoder.model.{i}.convtr.', cfg, ratio)
        i += 1
        for j in range(cfg['n_residual_layers']):
            x = resblock(x, sd, f'decoder.model.{i}.', cfg, cfg['dilation_base'] ** j)
            i += 1
    i += 1
    return conv(EO.elu(x), sd, f'decoder.model.{i}.conv.', cfg)


def preprocess(x, cfg):
    """EncodecModel.preprocess (audiocraft/models/encodec.py:186-196) = transformers EncodecModel._encode_frame's scale."""
    if not cfg.get('renormalize', False):
        return x, None
    scale = 1e-8 + x.mean(dim=1, keepdim=True).pow(2).mean(dim=2, keepdim=True).sqrt()
    return x / scale, scale.view(-1, 1)


def encode(x, sd, cfg, n_q):
    """One chunk: (codes [B, n_q, T], scale [B, 1] or None, latent)."""
    x, scale = preprocess(x.float(), cfg)
    lat = encode_latent(x, sd, cfg)
    return EO.rvq_encode(lat, EO.codebooks_of(sd, n_q)), scale, lat


def decode(codes, sd, cfg, scale=None):
    out = decode_latent(EO.rvq_decode(codes, EO.codebooks_of(sd, codes.shape[1])), sd, cfg)
    return out if scale is None else out * scale.view(-1, 1, 1)


def chunk_starts(length, chunk_length, stride):
    return list(range(0, length, stride))


def encode_chunks(x, sd, cfg, n_q, chunk_length, stride):
    """transformers EncodecModel.encode: chunks at offsets 0, stride, ... encoded independently, the last one's codes padded
    with zeros to the first one's frame count.  -> (codes [n, B, n_q, F], scales, last_frame_pad_length)."""
    codes, scales = [], []
    for o in chunk_starts(x.shape[-1], chunk_length, stride):
        c, s, _ = encode(x[..., o:o + chunk_length], sd, cfg, n_q)
        codes.append(c)
        scales.append(s)
    pad = codes[0].shape[-1] - codes[-1].shape[-1]
    codes[-1] = F.pad(codes[-1], (0, pad))
    return torch.stack(codes), scales, pad


def linear_overlap_add(frames, stride):
    """transformers EncodecModel._linear_overlap_add: triangle weights of the first frame's length, weighted sum over the
    overlapping frames divided by the summed weights."""
    total = stride * (len(frames) - 1) + frames[-1].shape[-1]
    n = frames[0].shape[-1]
    dt = frames[0].dtype
    t = torch.linspace(0, 1, n + 2, dtype=dt)[1:-1]
    weight = 0.5 - (t - 0.5).abs()
    out = torch.zeros(*frames[0].shape[:-1], total, dtype=dt)
    wsum = torch.zeros(total, dtype=dt)
    for i, f in enumerate(frames):
        o = i * stride
        out[..., o:o + f.shape[-1]] += weight[:f.shape[-1]] * f
        wsum[o:o + f.shape[-1]] += weight[:f.shape[-1]]
    return out / wsum


def decode_chunks(codes, scales, sd, cfg, stride, pad=0):
    frames = []
    for i in range(len(codes)):
        c = codes[i]
        if i == len(codes) - 1 and pad > 0:
            c = c[..., :-pad]
        frames.append(decode(c, sd, cfg, scales[i]))
    return linear_overlap_add(frames, stride)


def hf_48k_config(**over):
    """transformers' EncodecConfig of facebook/encodec_48khz (its config.json fields; the rest are EncodecConfig defaults)."""
    from transformers import EncodecConfig
    kw = dict(sampling_rate=48000, audio_channels=2, normalize=True, chunk_length_s=1.0, overlap=0.01,
              norm_type='time_group_norm', use_causal_conv=False, target_bandwidths=[3.0, 6.0, 12.0, 24.0])
    kw.update(over)
    return EncodecConfig(**kw)


def hf_48k_model(seed=0, **over):
    """transformers' 48 kHz EncodecModel with seeded weights: GroupNorm gamma / beta drawn around 1 / 0 (the default init
    leaves them at exactly 1 / 0, which would hide a transposed gamma or a dropped beta) and random codebooks."""
    import warnings
    from transformers import EncodecModel
    warnings.filterwarnings('ignore')
    torch.manual_seed(seed)
    hf = EncodecModel(hf_48k_config(**over)).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for k, v in hf.state_dict().items():
            if k.endswith('norm.weight'):
                v.copy_(1.0 + 0.2 * torch.randn(v.shape, generator=g))
            elif k.endswith('norm.bias'):
                v.copy_(0.1 * torch.randn(v.shape, generator=g))
            elif k.endswith('codebook.embed'):
                v.copy_(torch.randn(v.shape, generator=g) * 0.5)
    return hf
