"""CPU oracle for the EnCodec path: SEANet encoder/decoder + residual vector quantizer.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Plain fp32 torch ops on CPU; no reference
code is imported here, every function restates the algorithm and cites where it lives in the
reference (paths relative to the reference source tree).

Weights come in as a reference-layout ``state_dict`` (SURVEY.md section 8b):
  encoder.model.{i}.conv.conv.{weight_g,weight_v,bias}, encoder.model.{i}.block.{1,3}.conv.conv.*,
  encoder.model.{i}.lstm.{weight_ih_l0,...}, decoder.model.{i}.convtr.convtr.*,
  quantizer.vq.layers.{k}._codebook.embed
"""
import math
import typing as tp

import torch
import torch.nn.functional as F

DEFAULT_CFG = dict(
    channels=1, dimension=128, n_filters=32, n_residual_layers=1, ratios=[8, 5, 4, 2],
    kernel_size=7, last_kernel_size=7, residual_kernel_size=3, dilation_base=2, causal=False,
    pad_mode='reflect', compress=2, lstm=2, norm='weight_norm', trim_right_ratio=1.0,
    sample_rate=24000, n_q=8, bins=1024, renormalize=False,
)


def make_cfg(**over) -> dict:
    cfg = dict(DEFAULT_CFG)
    cfg.update(over)
    return cfg


# ----------------------------------------------------------------------------- padding rules

def extra_padding(length: int, k_eff: int, stride: int, padding_total: int) -> int:
    """Right padding so the last window is full. audiocraft/modules/conv.py:47-53."""
    n_frames = (length - k_eff + padding_total) / stride + 1
    ideal = (math.ceil(n_frames) - 1) * stride + (k_eff - padding_total)
    return ideal - length


def conv_paddings(length: int, kernel: int, stride: int, dilation: int, causal: bool) -> tp.Tuple[int, int]:
    """(left, right) padding applied by StreamableConv1d. audiocraft/modules/conv.py:185-200."""
    k_eff = (kernel - 1) * dilation + 1
    total = k_eff - stride
    extra = extra_padding(length, k_eff, stride, total)
    if causal:
        return total, extra
    right = total // 2
    return total - right, right + extra


def pad1d(x: torch.Tensor, left: int, right: int, mode: str) -> torch.Tensor:
    """Reflect pad that tolerates inputs shorter than the pad. audiocraft/modules/conv.py:71-88."""
    if mode != 'reflect':
        return F.pad(x, (left, right), mode)
    length = x.shape[-1]
    big = max(left, right)
    grow = 0
    if length <= big:
        grow = big - length + 1
        x = F.pad(x, (0, grow))
    y = F.pad(x, (left, right), 'reflect')
    return y[..., : y.shape[-1] - grow]


def fold_weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """w = g * v / ||v||, norm over every dim but 0 (torch.nn.utils.weight_norm, dim=0), as wrapped by
    audiocraft/modules/conv.py:21-30.  For ConvTranspose1d dim 0 is the INPUT channel."""
    n = v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (v.dim() - 1)))
    return v * (g / n)


def _conv_weight(sd: dict, prefix: str) -> tp.Tuple[torch.Tensor, torch.Tensor]:
    if prefix + 'weight_g' in sd:
        w = fold_weight_norm(sd[prefix + 'weight_g'].float(), sd[prefix + 'weight_v'].float())
    else:
        w = sd[prefix + 'weight'].float()
    return w, sd[prefix + 'bias'].float()


def sconv1d(x, w, b, stride=1, dilation=1, causal=False, pad_mode='reflect'):
    """StreamableConv1d.forward. audiocraft/modules/conv.py:185-201."""
    left, right = conv_paddings(x.shape[-1], w.shape[-1], stride, dilation, causal)
    return F.conv1d(pad1d(x, left, right, pad_mode), w, b, stride=stride, dilation=dilation)


def sconvtr1d(x, w, b, stride, causal=False, trim_right_ratio=1.0):
    """StreamableConvTranspose1d.forward: full transposed conv then trim the fixed padding.
    audiocraft/modules/conv.py:221-243."""
    k = w.shape[-1]
    total = k - stride
    y = F.conv_transpose1d(x, w, b, stride=stride)
    if causal:
        right = math.ceil(total * trim_right_ratio)
        left = total - right
    else:
        right = total // 2
        left = total - right
    return y[..., left: y.shape[-1] - right]


def elu(x):
    return F.elu(x, alpha=1.0)


def lstm_block(x: torch.Tensor, sd: dict, prefix: str, layers: int) -> torch.Tensor:
    """StreamableLSTM.forward: y = LSTM_layers(x) + x over the frame axis, conv layout in/out.
    audiocraft/modules/lstm.py:19-25 (nn.LSTM gate order i,f,g,o; zero initial state)."""
    seq = x.permute(2, 0, 1)  # [T, B, C]
    inp = seq
    for layer in range(layers):
        w_ih = sd[f'{prefix}weight_ih_l{layer}'].float()
        w_hh = sd[f'{prefix}weight_hh_l{layer}'].float()
        bias = sd[f'{prefix}bias_ih_l{layer}'].float() + sd[f'{prefix}bias_hh_l{layer}'].float()
        hid = w_hh.shape[1]
        h = torch.zeros(inp.shape[1], hid)
        c = torch.zeros(inp.shape[1], hid)
        gx = inp @ w_ih.t() + bias  # [T, B, 4H]
        outs = []
        for t in range(inp.shape[0]):
            gates = gx[t] + h @ w_hh.t()
            i, f, g, o = gates.split(hid, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            h = torch.sigmoid(o) * torch.tanh(c)
            outs.append(h)
        inp = torch.stack(outs)
    return (inp + seq).permute(1, 2, 0)


# ----------------------------------------------------------------------------- SEANet

def _resblock(x, sd, prefix, cfg, dilation):
    """SEANetResnetBlock.forward with true skip: x + conv1(ELU(conv_k(ELU(x)))).
    audiocraft/modules/seanet.py:36-60."""
    w1, b1 = _conv_weight(sd, prefix + 'block.1.conv.conv.')
    w2, b2 = _conv_weight(sd, prefix + 'block.3.conv.conv.')
    y = sconv1d(elu(x), w1, b1, dilation=dilation, causal=cfg['causal'], pad_mode=cfg['pad_mode'])
    y = sconv1d(elu(y), w2, b2, causal=cfg['causal'], pad_mode=cfg['pad_mode'])
    if not cfg.get('true_skip', True):   # 1x1 conv shortcut instead of the identity (seanet.py:54-57)
        ws, bs = _conv_weight(sd, prefix + 'shortcut.conv.conv.')
        x = sconv1d(x, ws, bs, causal=cfg['causal'], pad_mode=cfg['pad_mode'])
    return x + y


def seanet_encode(x: torch.Tensor, sd: dict, cfg: dict, prefix: str = 'encoder.') -> torch.Tensor:
    """SEANetEncoder.forward, module indices as built at audiocraft/modules/seanet.py:113-150."""
    kw = dict(causal=cfg['causal'], pad_mode=cfg['pad_mode'])
    i = 0
    w, b = _conv_weight(sd, f'{prefix}model.{i}.conv.conv.')
    x = sconv1d(x, w, b, **kw)
    i += 1
    for ratio in reversed(cfg['ratios']):
        for j in range(cfg['n_residual_layers']):
            x = _resblock(x, sd, f'{prefix}model.{i}.', cfg, cfg['dilation_base'] ** j)
            i += 1
        i += 1  # the ELU module
        w, b = _conv_weight(sd, f'{prefix}model.{i}.conv.conv.')
        x = sconv1d(elu(x), w, b, stride=ratio, **kw)
        i += 1
    if cfg['lstm']:
        x = lstm_block(x, sd, f'{prefix}model.{i}.lstm.', cfg['lstm'])
        i += 1
    i += 1  # ELU
    w, b = _conv_weight(sd, f'{prefix}model.{i}.conv.conv.')
    return sconv1d(elu(x), w, b, **kw)


def seanet_decode(z: torch.Tensor, sd: dict, cfg: dict, prefix: str = 'decoder.') -> torch.Tensor:
    """SEANetDecoder.forward, module indices as built at audiocraft/modules/seanet.py:207-254."""
    kw = dict(causal=cfg['causal'], pad_mode=cfg['pad_mode'])
    i = 0
    w, b = _conv_weight(sd, f'{prefix}model.{i}.conv.conv.')
    x = sconv1d(z, w, b, **kw)
    i += 1
    if cfg['lstm']:
        x = lstm_block(x, sd, f'{prefix}model.{i}.lstm.', cfg['lstm'])
        i += 1
    for ratio in cfg['ratios']:
        i += 1  # ELU
        w, b = _conv_weight(sd, f'{prefix}model.{i}.convtr.convtr.')
        x = sconvtr1d(elu(x), w, b, ratio, causal=cfg['causal'], trim_right_ratio=cfg['trim_right_ratio'])
        i += 1
        for j in range(cfg['n_residual_layers']):
            x = _resblock(x, sd, f'{prefix}model.{i}.', cfg, cfg['dilation_base'] ** j)
            i += 1
    i += 1  # ELU
    w, b = _conv_weight(sd, f'{prefix}model.{i}.conv.conv.')
    return sconv1d(elu(x), w, b, **kw)


# ----------------------------------------------------------------------------- RVQ

def codebooks_of(sd: dict, n_q: int) -> tp.List[torch.Tensor]:
    return [sd[f'quantizer.vq.layers.{k}._codebook.embed'].float() for k in range(n_q)]


def vq_nearest(x: torch.Tensor, embed: torch.Tensor) -> torch.Tensor:
    """EuclideanCodebook.quantize: argmax_j -(|x|^2 - 2 x.e_j + |e_j|^2), first max wins.
    audiocraft/quantization/core_vq.py:164-172.  x [N, D], embed [bins, D]."""
    e = embed.t()
    dist = -(x.pow(2).sum(1, keepdim=True) - 2 * x @ e + e.pow(2).sum(0, keepdim=True))
    return dist.max(dim=-1).indices


def rvq_encode(z: torch.Tensor, codebooks: tp.Sequence[torch.Tensor], return_margin: bool = False):
    """ResidualVectorQuantization.encode + ResidualVectorQuantizer.encode transpose.
    audiocraft/quantization/core_vq.py:386-396, vq.py:87-96.  z [B, D, T] -> codes [B, K, T] int64.
    With return_margin also returns, per code, the gap between the best and second-best score
    (used by the parity tests to tell a genuine mismatch from a floating-point near-tie)."""
    B, D, T = z.shape
    res = z.permute(0, 2, 1).reshape(B * T, D).clone()
    out, margins = [], []
    for embed in codebooks:
        if return_margin:
            e = embed.t()
            dist = -(res.pow(2).sum(1, keepdim=True) - 2 * res @ e + e.pow(2).sum(0, keepdim=True))
            top2 = dist.topk(2, dim=-1).values
            margins.append((top2[:, 0] - top2[:, 1]).reshape(B, T))
            idx = dist.max(dim=-1).indices
        else:
            idx = vq_nearest(res, embed)
        res = res - F.embedding(idx, embed)
        out.append(idx.reshape(B, T))
    codes = torch.stack(out, dim=1)
    if return_margin:
        return codes, torch.stack(margins, dim=1)
    return codes


def rvq_decode(codes: torch.Tensor, codebooks: tp.Sequence[torch.Tensor]) -> torch.Tensor:
    """ResidualVectorQuantization.decode: sum_k embed_k[codes[:,k]] -> [B, D, T].
    audiocraft/quantization/core_vq.py:398-404, vq.py:98-103."""
    acc = torch.zeros(())
    for k in range(codes.shape[1]):
        acc = acc + F.embedding(codes[:, k], codebooks[k])  # [B, T, D]
    return acc.permute(0, 2, 1)


# ----------------------------------------------------------------------------- model glue

class EncodecOracle:
    """EncodecModel.encode/decode/decode_latent. audiocraft/models/encodec.py:186-259."""

    def __init__(self, state_dict: dict, cfg: dict):
        self.sd = {k: v.detach().cpu() for k, v in state_dict.items()}
        self.cfg = cfg
        self.n_q = cfg['n_q']

    def preprocess(self, x):
        if not self.cfg.get('renormalize', False):
            return x, None
        mono = x.mean(dim=1, keepdim=True)
        scale = 1e-8 + mono.pow(2).mean(dim=2, keepdim=True).sqrt()
        return x / scale, scale.view(-1, 1)

    def encode_latent(self, x):
        return seanet_encode(x.float(), self.sd, self.cfg)

    def encode(self, x):
        x, scale = self.preprocess(x.float())
        emb = seanet_encode(x, self.sd, self.cfg)
        return rvq_encode(emb, codebooks_of(self.sd, self.n_q)), scale

    def decode_latent(self, codes):
        return rvq_decode(codes, codebooks_of(self.sd, codes.shape[1]))

    def decode(self, codes, scale=None):
        out = seanet_decode(self.decode_latent(codes), self.sd, self.cfg)
        if scale is not None:
            out = out * scale.view(-1, 1, 1)
        return out
