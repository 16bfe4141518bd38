"""T5 text encoder on the device: a local Hugging Face T5 directory run by ``acb_t5_encode`` (csrc/t5.cu).

The reference's ``T5Conditioner`` (conditioners.py:422-515) runs transformers' ``T5EncoderModel`` in fp32 and applies
``output_proj`` and the attention mask.  Here the weights of a local directory in Hugging Face layout (``config.json``,
``model.safetensors`` or ``pytorch_model.bin``, ``spiece.model``) are read once, kept fp32 on the device, and the whole
encoder plus the projection runs in the package's kernels.  Tokenization uses transformers' own ``T5Tokenizer`` on the host
(imported lazily), so ids and masks are the reference's by construction.  Nothing here resolves a hub name.
"""
import json
import math
import os
import typing as tp

import torch

from . import _lib

import ctypes as C


def read_config(path: str) -> dict:
    """The fields of a T5 ``config.json`` the encoder needs; variants the kernels do not implement raise."""
    with open(os.path.join(path, 'config.json')) as fh:
        raw = json.load(fh)
    ffp = raw.get('feed_forward_proj', 'relu')
    if ffp != 'relu':
        raise NotImplementedError(f"T5 feed_forward_proj '{ffp}' is not built (only 'relu', the original t5-small / base / "
                                  "large; flan-t5 uses a gated GELU)")
    cfg = dict(d_model=int(raw['d_model']), d_kv=int(raw['d_kv']), num_heads=int(raw['num_heads']),
               num_layers=int(raw['num_layers']), d_ff=int(raw['d_ff']), vocab_size=int(raw['vocab_size']),
               num_buckets=int(raw.get('relative_attention_num_buckets', 32)),
               max_distance=int(raw.get('relative_attention_max_distance', 128)),
               eps=float(raw.get('layer_norm_epsilon', 1e-6)))
    if cfg['d_kv'] != 64:
        raise NotImplementedError(f"T5 d_kv {cfg['d_kv']} is not built (the attention kernel has head_dim 64; "
                                  "t5-3b / t5-11b use 128)")
    if cfg['num_heads'] * cfg['d_kv'] != cfg['d_model'] or cfg['d_model'] % 64 or cfg['d_model'] > 2048:
        raise NotImplementedError(f"T5 d_model {cfg['d_model']} with {cfg['num_heads']} heads is not built "
                                  "(needs num_heads * 64 == d_model <= 2048)")
    return cfg


def read_state_dict(path: str) -> tp.Dict[str, torch.Tensor]:
    """``model.safetensors`` if present, else ``pytorch_model.bin`` (loaded with weights_only=True)."""
    st = os.path.join(path, 'model.safetensors')
    if os.path.exists(st):
        from safetensors.torch import load_file
        return load_file(st)
    binf = os.path.join(path, 'pytorch_model.bin')
    if os.path.exists(binf):
        return torch.load(binf, map_location='cpu', weights_only=True)
    raise FileNotFoundError(f"{path}: neither model.safetensors nor pytorch_model.bin")


def map_weights(sd: tp.Dict[str, torch.Tensor], cfg: dict) -> tp.Dict[str, torch.Tensor]:
    """transformers' T5 keys -> the stacked fp32 CPU tensors of acb_t5_weights (without the conditioner's projection)."""
    def get(k):
        if k not in sd:
            raise KeyError(f"T5 state dict has no '{k}'")
        return sd[k].float()
    L = cfg['num_layers']
    blk = 'encoder.block.{}.layer.{}.'
    w = {'shared': get('shared.weight')}
    w['w_qkv'] = torch.stack([torch.cat([get(blk.format(i, 0) + f'SelfAttention.{n}.weight') for n in 'qkv']) for i in range(L)])
    w['w_o'] = torch.stack([get(blk.format(i, 0) + 'SelfAttention.o.weight') for i in range(L)])
    w['w_i'] = torch.stack([get(blk.format(i, 1) + 'DenseReluDense.wi.weight') for i in range(L)])
    w['w_fo'] = torch.stack([get(blk.format(i, 1) + 'DenseReluDense.wo.weight') for i in range(L)])
    w['ln'] = torch.stack([torch.stack([get(blk.format(i, j) + 'layer_norm.weight') for j in (0, 1)]) for i in range(L)])
    w['final_ln'] = get('encoder.final_layer_norm.weight')
    w['rel_bias'] = get(blk.format(0, 0) + 'SelfAttention.relative_attention_bias.weight')
    d, ff, H = cfg['d_model'], cfg['d_ff'], cfg['num_heads']
    want = dict(shared=(cfg['vocab_size'], d), w_qkv=(L, 3 * d, d), w_o=(L, d, d), w_i=(L, ff, d), w_fo=(L, d, ff),
                ln=(L, 2, d), final_ln=(d,), rel_bias=(cfg['num_buckets'], H))
    for k, shape in want.items():
        if tuple(w[k].shape) != shape:
            raise ValueError(f"T5 weight {k}: shape {tuple(w[k].shape)}, config.json implies {shape}")
    return w


def relative_position_buckets(seq_len: int, num_buckets: int, max_distance: int) -> torch.Tensor:
    """int32 [2 seq_len - 1]: entry r is the bidirectional bucket of relative position r - (seq_len - 1) (key minus query),
    by the fp32 torch arithmetic of transformers' T5Attention._relative_position_bucket."""
    rel = torch.arange(-(seq_len - 1), seq_len, dtype=torch.long)
    nb = num_buckets // 2
    out = (rel > 0).to(torch.long) * nb
    n = torch.abs(rel)
    max_exact = nb // 2
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(max_distance / max_exact) * (nb - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, nb - 1))
    return (out + torch.where(n < max_exact, n, large)).to(torch.int32)


def round_tf32(t: torch.Tensor) -> torch.Tensor:
    """fp32 values rounded to the nearest TF32 value (10-bit mantissa, ties to even), as fp32.  The TF32 tensor core
    truncates the 13 low mantissa bits of an fp32 operand; weights rounded once here carry half that error."""
    b = t.float().contiguous().view(torch.int32)
    b = (b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF
    return b.view(torch.float32)


def load_tokenizer(path: str):
    """transformers' T5Tokenizer from the local directory (never the hub)."""
    from transformers import T5Tokenizer
    return T5Tokenizer.from_pretrained(path, local_files_only=True)


class T5Encoder:
    """The frozen T5 encoder of a local directory, fp32 on the device.  ``encode(ids, mask, proj_w, proj_b)`` returns
    ``(output_proj(T5(ids)) * mask, hidden or None)`` computed by acb_t5_encode."""

    def __init__(self, path: str, device='cuda'):
        self.path = path
        self.device = _lib.require_cuda(device)
        self.cfg = read_config(path)
        self._lib = _lib.lib()
        w = map_weights(read_state_dict(path), self.cfg)
        gemm = ('w_qkv', 'w_o', 'w_i', 'w_fo')   # GEMM operands; the embedding, norms and bias table stay exact
        self.w = {k: (round_tf32(v) if k in gemm else v).to(self.device).contiguous() for k, v in w.items()}
        self._buckets: tp.Dict[int, torch.Tensor] = {}

    @property
    def d_model(self) -> int:
        return self.cfg['d_model']

    def buckets(self, seq_len: int) -> torch.Tensor:
        if seq_len not in self._buckets:
            self._buckets[seq_len] = relative_position_buckets(
                seq_len, self.cfg['num_buckets'], self.cfg['max_distance']).to(self.device)
        return self._buckets[seq_len]

    def _abi(self, out_dim: int, proj_w: torch.Tensor, proj_b: torch.Tensor):
        c = self.cfg
        conf = _lib.T5Config(c['d_model'], c['d_kv'], c['num_heads'], c['num_layers'], c['d_ff'], c['vocab_size'],
                             c['num_buckets'], out_dim, c['eps'])
        w = self.w
        wts = _lib.T5Weights(*[_lib.ptr(t) for t in (w['shared'], w['w_qkv'], w['w_o'], w['w_i'], w['w_fo'], w['ln'],
                                                      w['final_ln'], w['rel_bias'], proj_w, proj_b)])
        return conf, wts

    @torch.no_grad()
    def encode(self, ids: torch.Tensor, mask: torch.Tensor, proj_w: torch.Tensor, proj_b: torch.Tensor,
               return_hidden: bool = False):
        B, T = ids.shape
        if int(ids.min()) < 0 or int(ids.max()) >= self.cfg['vocab_size']:
            raise ValueError(f"token ids must lie in [0, {self.cfg['vocab_size']})")
        ids = ids.to(self.device, torch.long).contiguous()
        mask = mask.to(self.device, torch.long).contiguous()
        proj_w = round_tf32(proj_w.detach().to(self.device, torch.float32))
        proj_b = proj_b.to(self.device, torch.float32).contiguous()
        out_dim = proj_w.shape[0]
        assert proj_w.shape == (out_dim, self.d_model) and proj_b.shape == (out_dim,)
        conf, wts = self._abi(out_dim, proj_w, proj_b)
        with torch.cuda.device(self.device):
            nbytes = self._lib.acb_t5_workspace_bytes(C.byref(conf), B, T)
            if nbytes < 0:
                _lib.check(int(nbytes), 't5_workspace_bytes')
            ws = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=self.device)
            out = torch.empty((B, T, out_dim), dtype=torch.float32, device=self.device)
            hidden = torch.empty((B, T, self.d_model), dtype=torch.float32, device=self.device) if return_hidden else None
            _lib.check(self._lib.acb_t5_encode(C.byref(conf), C.byref(wts), _lib.ptr(ids), _lib.ptr(mask),
                                               _lib.ptr(self.buckets(T)), B, T, _lib.ptr(out), _lib.ptr(hidden),
                                               _lib.ptr(ws), int(nbytes), _lib.stream()), 't5_encode')
        return out, hidden
