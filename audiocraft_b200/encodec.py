"""EnCodec on H100: host-side mirror of ``audiocraft.models.encodec`` over the C-ABI kernels.

``CompressionModel`` keeps the reference's abstract surface (audiocraft/models/encodec.py:28-122);
``EncodecModel`` keeps ``encode / decode / decode_latent / preprocess / postprocess`` and the properties
(audiocraft/models/encodec.py:125-259) but is built from a reference-layout ``state_dict`` + hyper-parameters
instead of nn.Modules: weight-norm is folded once at load on the GPU, conv weights are re-packed tap-major,
and every layer is one fused kernel (padding, ELU, bias, residual, trim inside).

PyTorch here is plumbing only (device memory, streams).  There is no CPU path: without the CUDA library
or a GPU, construction raises.
"""
import copy
import math
import os
import typing as tp
from abc import ABC, abstractmethod

import torch

from . import _lib
from .synth import ENCODEC_CONFIGS, encodec_hop, encodec_layers


class CompressionModel(ABC):
    """Same abstract API as audiocraft.models.encodec.CompressionModel (encodec.py:28-122)."""

    @abstractmethod
    def forward(self, x: torch.Tensor): ...

    @abstractmethod
    def encode(self, x: torch.Tensor) -> tp.Tuple[torch.Tensor, tp.Optional[torch.Tensor]]: ...

    @abstractmethod
    def decode(self, codes: torch.Tensor, scale: tp.Optional[torch.Tensor] = None): ...

    @abstractmethod
    def decode_latent(self, codes: torch.Tensor): ...

    @property
    @abstractmethod
    def channels(self) -> int: ...

    @property
    @abstractmethod
    def frame_rate(self) -> float: ...

    @property
    @abstractmethod
    def sample_rate(self) -> int: ...

    @property
    @abstractmethod
    def cardinality(self) -> int: ...

    @property
    @abstractmethod
    def num_codebooks(self) -> int: ...

    @property
    @abstractmethod
    def total_codebooks(self) -> int: ...

    @abstractmethod
    def set_num_codebooks(self, n: int): ...

    def eval(self):
        return self

    def __call__(self, x):
        return self.forward(x)

    @staticmethod
    def get_pretrained(name: str, device='cuda') -> 'CompressionModel':
        """The reference downloads checkpoints from the HF hub (encodec.py:87-122).  There is no network here:
        `name` may be a local checkpoint file in the reference's export format
        ({'best_state', 'xp.cfg'} -- audiocraft/utils/export.py:20-79), a local directory holding a transformers EnCodec
        snapshot (config.json + weights, what the reference reaches for `facebook/encodec_*`), or one of the synthetic
        architectures."""
        if os.path.isdir(name) and os.path.isfile(os.path.join(name, 'config.json')):
            return HFEncodecCompressionModel.from_pretrained_dir(name, device=device)
        from .loaders import load_compression_model
        return load_compression_model(name, device=device)


# ----------------------------------------------------------------------------- host-side padding rules

def extra_padding(length: int, k_eff: int, stride: int, padding_total: int) -> int:
    """get_extra_padding_for_conv1d, audiocraft/modules/conv.py:47-53."""
    n_frames = (length - k_eff + padding_total) / stride + 1
    return (math.ceil(n_frames) - 1) * stride + (k_eff - padding_total) - length


def conv_geometry(length: int, kernel: int, stride: int, dilation: int, causal: bool, reflect: bool):
    """(pad_left, t_virtual, t_out) of StreamableConv1d.forward for an input of `length` steps
    (audiocraft/modules/conv.py:185-200 + the short-input rule of pad1d :71-88)."""
    k_eff = (kernel - 1) * dilation + 1
    total = k_eff - stride
    extra = extra_padding(length, k_eff, stride, total)
    if causal:
        left, right = total, extra
    else:
        right = total // 2
        left = total - right
        right += extra
    t_virtual = length
    if reflect and length <= max(left, right):
        t_virtual = length + (max(left, right) - length + 1)
    t_out = (length + left + right - k_eff) // stride + 1
    return left, t_virtual, t_out


def convtr_geometry(length: int, kernel: int, stride: int, causal: bool, trim_right_ratio: float):
    """(trim_left, t_out) of StreamableConvTranspose1d.forward (audiocraft/modules/conv.py:221-243)."""
    total = kernel - stride
    if causal:
        right = math.ceil(total * trim_right_ratio)
        left = total - right
    else:
        right = total // 2
        left = total - right
    t_full = (length - 1) * stride + kernel
    return left, t_full - left - right


def tf32_round(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> nearest tf32-representable fp32 (10-bit mantissa), ties away from zero: what `cvt.rna.tf32.f32` returns."""
    bits = x.contiguous().view(torch.int32)
    return ((bits + 0x1000) & -8192).view(torch.float32)


def pack_conv_t6(w: torch.Tensor, tile: int) -> torch.Tensor:
    """Weights [c_out][c_in][K] (weight-norm folded) -> the operand layout of the experimental `acb_conv1d_t6`:
    two tf32 terms (hi, lo = tf32(w - hi)) as [c_out/tile][c_in/8][K][term][2][tile][4]: per (tile, 8-channel group, tap)
    a K-major wgmma B operand (rows = output channels at 16 B pitch, two 4-channel chunks tile*16 B apart)."""
    co, ci, K = w.shape
    assert co % tile == 0 and ci % 8 == 0, (w.shape, tile)
    hi = tf32_round(w.float())
    lo = tf32_round(w.float() - hi)
    t = torch.stack([hi, lo]).view(2, co // tile, tile, ci // 8, 2, 4, K)   # term, tile, n, cg, c, j, k
    return t.permute(1, 3, 6, 0, 4, 2, 5).contiguous()                      # tile, cg, k, term, c, n, j


def check_norm(cfg: dict) -> float:
    """The conv normalisations the kernels run (CONV_NORMALIZATIONS, audiocraft/modules/conv.py:17-42): 'weight_norm'
    (folded at load), 'none', and 'time_group_norm' = GroupNorm(1, C) after every convolution, which the reference refuses
    on a causal model.  Anything else raises here rather than running the codec without its norm.  Returns the GroupNorm eps."""
    norm = cfg.get('norm', 'weight_norm')
    params = dict(cfg.get('norm_params') or {})
    if norm not in ('weight_norm', 'none', 'time_group_norm'):
        raise NotImplementedError(f"conv norm '{norm}' is not built (weight_norm, none and time_group_norm are)")
    if norm == 'time_group_norm' and cfg['causal']:
        raise ValueError("GroupNorm doesn't support causal evaluation.")   # get_norm_module, conv.py:37-38
    if set(params) - {'eps'}:
        raise NotImplementedError(f"norm_params {sorted(set(params) - {'eps'})} are not built (only eps)")
    return float(params.get('eps', 1e-5))


class EncodecModel(CompressionModel):
    """EnCodec (SEANet + RVQ) on H100 behind the reference's ``EncodecModel`` API."""

    def __init__(self, state_dict: tp.Dict[str, torch.Tensor], cfg: dict, device='cuda',
                 encoder_precision: str = 'fp32_tc', decoder_precision: str = 'tf32x3'):
        """encoder_precision / decoder_precision:
          'fp32'         every convolution on fp32 FMA;
          'fp32_tc'      (encoder default) fp32 ACCURACY on the tensor cores: layers with kernel > 1 and >= 128 output channels
                         run `acb_conv1d_t6` (wgmma, 3xTF32 operand split, the tensor-core accumulator flushed into fp32 registers
                         every 8 input channels), the rest fp32 FMA.  RVQ indices equal the fp32 reference's on the 24 / 32 kHz
                         goldens (tests/test_gpu_fullsize.py);
                         Residual blocks with the identity skip at 64 / 128 / 256 channels run as ONE kernel (`acb_resblock`, both
                         operands split into two fp16 terms = 22 mantissa bits, tensor-core accumulation runs cut every 48 / 16
                         reduction rows) in every precision except 'fp32'; the LSTM's recurrent step uses the same split;
          'tf32x3_flush' the same kernel on every layer it supports (slower on 1x1 convolutions; kept for tests);
          'tf32x3'       (decoder default, NOT fp32-exact) wgmma 3xTF32 without flushes: the decoder's output is a waveform
                         checked to a tolerance of 1e-4 (DESIGN.md section 4); as an encoder mode its latents move by 1.5e-4."""
        self._gn_eps = check_norm(cfg)
        self.device = _lib.require_cuda(device)
        prec = {'fp32': _lib.CONV_FP32, 'tf32x3': _lib.CONV_TF32X3, 'tf32x3_mmasync': _lib.CONV_TF32X3_MMASYNC,
                'tf32x3_flush': _lib.CONV_T6_FLUSH, 'fp32_tc': _lib.CONV_T6_AUTO}
        self._enc_prec, self._dec_prec = prec[encoder_precision], prec[decoder_precision]
        self._want_t6 = bool({_lib.CONV_T6_FLUSH, _lib.CONV_T6_AUTO} & {self._enc_prec, self._dec_prec})
        # the LSTM input projections (one 1x1 conv per layer) always run on the tensor cores: measured 3.9e-6 vs 3.6e-6 latent
        # error for the otherwise-fp32 encoder (the tensor-core error of the conv stack comes from its long reductions)
        self._lstm_prec = _lib.CONV_TF32X3
        import os as _os
        self._fuse_blocks = _os.environ.get('ACB_ENCODEC_FUSED_BLOCKS', '1') != '0'   # acb_resblock for the residual blocks it takes
        self._lib = _lib.lib()
        self.cfg = dict(cfg)
        self._channels = cfg['channels']
        self._sample_rate = cfg['sample_rate']
        self._frame_rate = cfg['sample_rate'] / encodec_hop(cfg)
        self.causal = cfg['causal']
        self.renormalize = cfg.get('renormalize', False)
        if self.causal:
            assert not self.renormalize, 'Causal model does not support renormalize'  # encodec.py:163-166
        self.max_n_q = cfg['n_q']
        self.n_q = cfg['n_q']
        self.bins = cfg['bins']
        self.dimension = cfg['dimension']
        self.reflect = 1 if cfg['pad_mode'] == 'reflect' else 0
        assert cfg['pad_mode'] in ('reflect', 'constant', 'zeros'), cfg['pad_mode']
        self.launches = 0
        plan = encodec_layers(cfg)
        with torch.cuda.device(self.device):
            self.enc = [self._prepare(layer, state_dict) for layer in plan['encoder']]
            self.dec = [self._prepare(layer, state_dict) for layer in plan['decoder']]
            cb = torch.stack([state_dict[f'quantizer.vq.layers.{k}._codebook.embed'].float()
                              for k in range(self.max_n_q)]).to(self.device).contiguous()
            self.codebooks = cb                                        # [n_q][bins][D]
            self.cb_sqnorm = cb.pow(2).sum(-1).contiguous()            # |e_j|^2, core_vq.py:169
            torch.cuda.synchronize(self.device)

    # ------------------------------------------------------------------ weight preparation (once)
    def _fold(self, sd, prefix):
        if prefix + 'weight_g' in sd:
            v = sd[prefix + 'weight_v'].to(self.device, torch.float32).contiguous()
            g = sd[prefix + 'weight_g'].to(self.device, torch.float32).contiguous()
            w = torch.empty_like(v)
            _lib.check(self._lib.acb_weight_norm_fold(_lib.ptr(v), _lib.ptr(g), _lib.ptr(w), v.shape[0],
                                                      v[0].numel(), _lib.stream()), 'weight_norm_fold')
            return w
        return sd[prefix + 'weight'].to(self.device, torch.float32).contiguous()

    def _prepare(self, layer: dict, sd) -> dict:
        out = dict(layer)
        p = layer['prefix']
        if layer['kind'] in ('conv', 'convtr'):
            # NormConv1d / NormConvTranspose1d hold the GroupNorm next to the conv (modules/conv.py:91-137): `...conv.norm.*`.
            # Read per layer from the weights, so blocks the reference builds with norm='none' (disable_norm_outer_blocks) have none
            n = p.rsplit('.', 2)[0] + '.norm.'
            out['gn'] = n + 'weight' in sd
            if out['gn']:
                out['gn_g'] = sd[n + 'weight'].to(self.device, torch.float32).contiguous()
                out['gn_b'] = sd[n + 'bias'].to(self.device, torch.float32).contiguous()
        if layer['kind'] == 'conv':
            w = self._fold(sd, p)                                       # [Cout][Cin][K]
            out['w'] = w.permute(1, 2, 0).reshape(-1, w.shape[0]).contiguous()   # [Cin*K][Cout]
            out['b'] = sd[p + 'bias'].to(self.device, torch.float32).contiguous()
            tile = int(self._lib.acb_conv1d_t6_tile(w.shape[0])) if self._want_t6 else 0
            if tile and w.shape[1] % 8 == 0:
                out['w6'] = pack_conv_t6(w, tile)
        elif layer['kind'] == 'convtr':
            w = self._fold(sd, p)                                       # [Cin][Cout][K]
            out['w'] = w.permute(0, 2, 1).contiguous()                  # [Cin][K][Cout]
            cin, cout, k = w.shape
            S = layer['stride']
            # GEMM operand of the tensor-core path: [2*Cin][Cout*S], row (ci, k'), column co*S + ph, value w[ci][co][ph + (1-k')*S]
            out['w_gemm'] = w.view(cin, cout, 2, S).flip(2).permute(0, 2, 1, 3).reshape(cin * 2, cout * S).contiguous()
            out['b'] = sd[p + 'bias'].to(self.device, torch.float32).contiguous()
        else:
            out['w_ih'], out['w_hh'], out['bias'] = [], [], []
            for n in range(layer['layers']):
                w_ih = sd[f'{p}weight_ih_l{n}'].to(self.device, torch.float32)
                out['w_ih'].append(w_ih.t().contiguous())              # 1x1 conv packing [H][4H]
                out['w_hh'].append(sd[f'{p}weight_hh_l{n}'].to(self.device, torch.float32).contiguous())
                out['bias'].append((sd[f'{p}bias_ih_l{n}'].float() + sd[f'{p}bias_hh_l{n}'].float())
                                   .to(self.device).contiguous())
        return out

    # ------------------------------------------------------------------ layer launches
    def _conv(self, x, L, w=None, b=None, res=None, k=None, stride=None, dilation=None, elu=None, cout=None,
              prec=0, valid=False):
        """valid=True: no padding, the outputs whose window lies inside x (a streaming window, audiocraft_b200/streaming.py)."""
        B, cin, T = x.shape
        k = L['k'] if k is None else k
        stride = L['stride'] if stride is None else stride
        dilation = L['dilation'] if dilation is None else dilation
        cout = L['cout'] if cout is None else cout
        if valid:
            left, t_virt, t_out = 0, T, (T - (k - 1) * dilation - 1) // stride + 1
        else:
            left, t_virt, t_out = conv_geometry(T, k, stride, dilation, self.causal, bool(self.reflect))
        y = torch.empty((B, cout, t_out), device=x.device, dtype=torch.float32)
        if prec == _lib.CONV_T6_AUTO:
            # the implicit-GEMM tensor-core kernel is for k > 1 with >= 128 output channels: a 1x1 convolution gives it too little
            # reduction per staged slab (a routing choice made on the previous GPU generation, not re-measured per layer on the H100)
            prec = _lib.CONV_T6_FLUSH if (k > 1 and cout >= 128) else _lib.CONV_FP32
        if prec == _lib.CONV_T6_FLUSH:
            if w is None and 'w6' in L and cout == L['cout']:
                _lib.check(self._lib.acb_conv1d_t6(_lib.ptr(x), _lib.ptr(L['w6']), _lib.ptr(L['b'] if b is None else b),
                                                   _lib.ptr(res), _lib.ptr(y), B, cin, cout, T, t_virt, t_out, k, stride,
                                                   dilation, left, self.reflect, int(L['elu'] if elu is None else elu),
                                                   _lib.stream()), 'conv1d_t6')
                self.launches += 1
                return y
            prec = _lib.CONV_FP32          # layers the implicit-GEMM kernel does not take keep fp32 accuracy on the FMA path
        _lib.check(self._lib.acb_conv1d(_lib.ptr(x), _lib.ptr(L['w'] if w is None else w),
                                        _lib.ptr(L['b'] if b is None else b), _lib.ptr(res), _lib.ptr(y),
                                        B, cin, cout, T, t_virt, t_out, k, stride, dilation, left, self.reflect,
                                        int(L['elu'] if elu is None else elu), prec, _lib.stream()), 'conv1d')
        self.launches += 1
        return y

    def _convtr(self, x, L, prec=0, trim=True, window=None):
        """trim=False: the full transposed-conv output (the GroupNorm statistics cover the steps the trim drops).
        window=(trim_left, t_out): that range of the full output (a streaming window)."""
        B, cin, T = x.shape
        trim_left, t_out = convtr_geometry(T, L['k'], L['stride'], self.causal, self.cfg['trim_right_ratio'])
        if not trim:
            trim_left, t_out = 0, (T - 1) * L['stride'] + L['k']
        if window is not None:
            trim_left, t_out = window
        y = torch.empty((B, L['cout'], t_out), device=x.device, dtype=torch.float32)
        if prec in (_lib.CONV_T6_FLUSH, _lib.CONV_T6_AUTO):
            prec = _lib.CONV_TF32X3        # transposed convs have no implicit-GEMM variant yet
        _lib.check(self._lib.acb_convtr1d(_lib.ptr(x), _lib.ptr(L['w']), _lib.ptr(L['w_gemm']), _lib.ptr(L['b']),
                                          _lib.ptr(y), B, cin, L['cout'], T, t_out, L['k'], L['stride'], trim_left,
                                          int(L['elu']), prec, _lib.stream()), 'convtr1d')
        self.launches += 1
        return y

    def _lstm(self, x, L, prec=0, state=None):
        """y = LSTM(x) + x over frames (audiocraft/modules/lstm.py:19-25): per layer one 1x1 conv for the input
        half of the gates, then the persistent recurrent kernel.  state: per-layer ([B, H], [B, H]) (h, c) to start from,
        advanced in place (acb_lstm_recurrent_carry)."""
        B, H, T = x.shape
        ws = torch.empty(int(self._lib.acb_lstm_state_bytes(B, H)) // 4, device=x.device, dtype=torch.float32)
        inp = x
        n_layers = len(L['w_hh'])
        for n in range(n_layers):
            gx = torch.empty((B, 4 * H, T), device=x.device, dtype=torch.float32)
            _lib.check(self._lib.acb_conv1d(_lib.ptr(inp), _lib.ptr(L['w_ih'][n]), _lib.ptr(L['bias'][n]), None,
                                            _lib.ptr(gx), B, H, 4 * H, T, T, T, 1, 1, 1, 0, 0, 0, prec, _lib.stream()),
                       'lstm input conv')
            y = torch.empty((B, H, T), device=x.device, dtype=torch.float32)
            skip = x if n == n_layers - 1 else None
            if state is not None:
                h, c = state[n]
                _lib.check(self._lib.acb_lstm_recurrent_carry(_lib.ptr(gx), _lib.ptr(L['w_hh'][n]), _lib.ptr(skip), _lib.ptr(y),
                                                              _lib.ptr(ws), _lib.ptr(h), _lib.ptr(c), B, H, T, _lib.stream()),
                           'lstm_recurrent_carry')
            else:
                _lib.check(self._lib.acb_lstm_recurrent(_lib.ptr(gx), _lib.ptr(L['w_hh'][n]), _lib.ptr(skip), _lib.ptr(y),
                                                        _lib.ptr(ws), B, H, T, _lib.stream()), 'lstm_recurrent')
            self.launches += 2
            inp = y
        return inp

    def _fused_block(self, layers, i, prec, T):
        """layers[i], layers[i+1] = the two convolutions of a SEANetResnetBlock with the identity skip that `acb_resblock` takes
        (64 / 128 / 256 channels, kernel sizes [3, 1]); every tensor-core precision uses it, 'fp32' (all-FMA) does not."""
        if prec == _lib.CONV_FP32 or not self._fuse_blocks or i + 1 >= len(layers) or T <= 2 * layers[i].get('dilation', 1):
            return False
        a, b = layers[i], layers[i + 1]
        return (a['kind'] == 'conv' and b['kind'] == 'conv' and a['res'] == 'in' and b['res'] == 'out' and a['stride'] == 1
                and b['k'] == 1 and b['stride'] == 1 and a['elu'] and b['elu'] and b['cout'] == 2 * a['cout']
                and bool(self._lib.acb_resblock_supported(b['cout'], a['k'], a['dilation'])))

    def _resblock(self, x, a, b, prec, pad_left=None):
        """pad_left given: zero padding of pad_left steps instead of the layer's own (a streaming window: the caller keeps the
        outputs that touched no padding)."""
        B, C, T = x.shape
        if 'w1p' not in a:   # [C*k][C/2] (row = ci*k + tap) -> [k][C][C/2]
            a['w1p'] = a['w'].view(C, a['k'], a['cout']).permute(1, 0, 2).contiguous()
        left, _, t_out = conv_geometry(T, a['k'], 1, a['dilation'], self.causal, bool(self.reflect))
        assert t_out == T
        reflect = self.reflect
        if pad_left is not None:
            left, reflect = pad_left, 0
        y = torch.empty_like(x)
        exact = int(prec in (_lib.CONV_T6_FLUSH, _lib.CONV_T6_AUTO))
        _lib.check(self._lib.acb_resblock(_lib.ptr(x), _lib.ptr(a['w1p']), _lib.ptr(a['b']), _lib.ptr(b['w']), _lib.ptr(b['b']),
                                          _lib.ptr(y), B, C, T, a['k'], a['dilation'], left, reflect, exact, _lib.stream()),
                   'resblock')
        self.launches += 1
        return y

    def _gn_stats(self, y):
        B, C, T = y.shape
        ws = torch.empty(int(self._lib.acb_groupnorm_workspace_bytes(B, C, T)), device=y.device, dtype=torch.uint8)
        st = torch.empty((B, 2), device=y.device, dtype=torch.float64)
        _lib.check(self._lib.acb_groupnorm_stats(_lib.ptr(y), _lib.ptr(ws), _lib.ptr(st), B, C, T, self._gn_eps, _lib.stream()),
                   'groupnorm_stats')
        self.launches += 2
        return st

    def _gn_apply(self, y, L, st, left=0, t_out=None, add=None):
        """GroupNorm of the conv output y (window [left, left + t_out)), plus `add`: a tensor (identity skip) or the
        (raw output, stats, layer) of a conv shortcut whose GroupNorm is applied here too."""
        B, C, T = y.shape
        t_out = T if t_out is None else t_out
        out = torch.empty((B, C, t_out), device=y.device, dtype=torch.float32)
        x2 = st2 = g2 = b2 = res = None
        if isinstance(add, tuple):
            x2, st2, L2 = add
            g2, b2 = L2['gn_g'], L2['gn_b']
        else:
            res = add
        _lib.check(self._lib.acb_groupnorm_apply(_lib.ptr(y), _lib.ptr(st), _lib.ptr(L['gn_g']), _lib.ptr(L['gn_b']), T, left,
                                                 _lib.ptr(x2), _lib.ptr(st2), _lib.ptr(g2), _lib.ptr(b2), _lib.ptr(res),
                                                 _lib.ptr(out), B, C, t_out, _lib.stream()), 'groupnorm_apply')
        self.launches += 1
        return out

    def _run_gn(self, x, layers, prec):
        """Layer order of a GroupNorm model: each conv runs without its residual epilogue, then the statistics of its output,
        then the apply kernel, which also adds the block's skip; the skip is added after both GroupNorms
        (SEANetResnetBlock.forward: shortcut(x) + block(x), modules/seanet.py:59-60)."""
        skip, have_shortcut = None, False
        for L in layers:
            if L['kind'] == 'lstm':
                x = self._lstm(x, L, prec=self._lstm_prec)
            elif L['kind'] == 'convtr':
                if not L['gn']:
                    x = self._convtr(x, L, prec=prec)
                    continue
                left, t_out = convtr_geometry(x.shape[-1], L['k'], L['stride'], self.causal, self.cfg['trim_right_ratio'])
                full = self._convtr(x, L, prec=prec, trim=False)
                x = self._gn_apply(full, L, self._gn_stats(full), left=left, t_out=t_out)
            elif L['res'] == 'shortcut':
                s = self._conv(x, L, prec=prec)
                skip = (s, self._gn_stats(s), L) if L['gn'] else s
                have_shortcut = True
            else:
                if L['res'] == 'in':
                    if not have_shortcut:
                        skip = x
                    have_shortcut = False
                add = skip if L['res'] == 'out' else None
                if not L['gn']:
                    assert not isinstance(add, tuple), 'a residual block with a GroupNorm on only one branch'
                    x = self._conv(x, L, res=add, prec=prec)
                    continue
                y = self._conv(x, L, prec=prec)
                x = self._gn_apply(y, L, self._gn_stats(y), add=add)
        return x

    def _run(self, x, layers, prec=0):
        if any(L.get('gn') for L in layers):
            return self._run_gn(x, layers, prec)
        skip, have_shortcut = None, False
        prof = getattr(self, '_profile', None)   # optional per-layer CUDA-event timing (profiles/perf_encodec.py)
        skip_next = False
        for i, L in enumerate(layers):
            if skip_next:                           # second convolution of a block the fused kernel already ran
                skip_next = False
                continue
            if not have_shortcut and self._fused_block(layers, i, prec, x.shape[-1]):
                if prof is not None:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    shape_in = tuple(x.shape)
                x = self._resblock(x, L, layers[i + 1], prec)
                skip_next = True
                if prof is not None:
                    e1.record()
                    prof.append((dict(L, prefix=L['prefix'] + ' [+1x1, fused block]'), shape_in, tuple(x.shape), e0, e1))
                continue
            if prof is not None:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                shape_in = tuple(x.shape)
            if L['kind'] == 'conv':
                if L['res'] == 'shortcut':          # skip = conv1x1(block input); the block input itself is unchanged
                    skip = self._conv(x, L, prec=prec)
                    have_shortcut = True
                    if prof is not None:
                        e1.record()
                        prof.append((L, shape_in, tuple(skip.shape), e0, e1))
                    continue
                if L['res'] == 'in':
                    if not have_shortcut:
                        skip = x
                    have_shortcut = False
                res = skip if L['res'] == 'out' else None
                x = self._conv(x, L, res=res, prec=prec)
            elif L['kind'] == 'convtr':
                x = self._convtr(x, L, prec=prec)
            else:
                x = self._lstm(x, L, prec=self._lstm_prec)
            if prof is not None:
                e1.record()
                prof.append((L, shape_in, tuple(x.shape), e0, e1))
        return x

    # ------------------------------------------------------------------ reference API
    @property
    def total_codebooks(self):
        return self.max_n_q

    @property
    def num_codebooks(self):
        return self.n_q

    def set_num_codebooks(self, n: int):
        assert n > 0 and n <= self.max_n_q   # vq.py:113-115
        self.n_q = n

    @property
    def cardinality(self):
        return self.bins

    @property
    def channels(self):
        return self._channels

    @property
    def frame_rate(self):
        return self._frame_rate

    @property
    def sample_rate(self):
        return self._sample_rate

    def preprocess(self, x):
        """encodec.py:186-196."""
        if self.renormalize:
            mono = x.mean(dim=1, keepdim=True)
            volume = mono.pow(2).mean(dim=2, keepdim=True).sqrt()
            scale = 1e-8 + volume
            return x / scale, scale.view(-1, 1)
        return x, None

    def postprocess(self, x, scale=None):
        if scale is not None:
            assert self.renormalize
            x = x * scale.view(-1, 1, 1)
        return x

    def _in(self, x):
        assert x.dim() == 3
        assert x.shape[1] == self._channels, f"expected {self._channels} channels, got {x.shape[1]}"
        return x.to(self.device, torch.float32).contiguous()

    def encode_latent(self, x):
        """SEANetEncoder.forward (audiocraft/modules/seanet.py:152-153) on pre-processed input."""
        with torch.cuda.device(self.device):
            return self._run(self._in(x), self.enc, self._enc_prec)

    def quantize(self, emb, n_q=None):
        """ResidualVectorQuantizer.encode (vq.py:87-96): latent [B,D,T] -> codes [B,n_q,T] int64 (n_q: default the active count)."""
        B, D, T = emb.shape
        n_q = self.n_q if n_q is None else n_q
        codes = torch.empty((B, n_q, T), device=emb.device, dtype=torch.int64)
        _lib.check(self._lib.acb_rvq_encode(_lib.ptr(emb.contiguous()), _lib.ptr(self.codebooks),
                                            _lib.ptr(self.cb_sqnorm), _lib.ptr(codes), B, D, T, n_q, self.bins,
                                            _lib.stream()), 'rvq_encode')
        self.launches += 1
        return codes

    def encode(self, x):
        """encodec.py:223-238."""
        with torch.cuda.device(self.device):
            x, scale = self.preprocess(self._in(x))
            emb = self._run(x.contiguous(), self.enc, self._enc_prec)
            return self.quantize(emb), scale

    def decode_latent(self, codes):
        """encodec.py:257-259 -> vq.py:98-103."""
        assert codes.dim() == 3
        with torch.cuda.device(self.device):
            codes = codes.to(self.device, torch.int64).contiguous()
            B, K, T = codes.shape
            assert K <= self.max_n_q
            # F.embedding in the reference (core_vq.py:177-179) raises on an out-of-range index; the gather kernel would
            # clamp, so refuse here (one host sync per decode)
            if codes.numel():
                lo, hi = int(codes.min()), int(codes.max())
                if lo < 0 or hi >= self.bins:
                    raise IndexError(f"codes out of range [0, {self.bins}): min {lo}, max {hi}")
            out = torch.empty((B, self.dimension, T), device=self.device, dtype=torch.float32)
            _lib.check(self._lib.acb_rvq_decode(_lib.ptr(codes), _lib.ptr(self.codebooks), _lib.ptr(out), B,
                                                self.dimension, T, K, self.bins, _lib.stream()), 'rvq_decode')
            self.launches += 1
            return out

    def decode(self, codes, scale=None):
        """encodec.py:240-255; like the reference the output keeps the decoder's extra padding."""
        with torch.cuda.device(self.device):
            out = self._run(self.decode_latent(codes), self.dec, self._dec_prec)
            return self.postprocess(out, scale)

    def stream_decoder(self, batch: int, scale=None) -> 'EncodecStreamDecoder':
        """A stateful decoder for codes that arrive in pieces: `push(codes [B, K, n])` returns the samples no later frame can
        change, `flush()` the rest, and their concatenation is `decode(all codes)` (same length).  Renormalisation scales are not
        part of MusicGen decoding and are refused; GroupNorm codecs are refused because their statistics span the whole item."""
        if self.cfg.get('norm') == 'time_group_norm':
            raise NotImplementedError("streaming decode of a GroupNorm codec (norm: time_group_norm) is not built: its "
                                      "statistics span the whole item")
        if scale is not None:
            raise NotImplementedError("streaming decode with a renormalisation scale is not built (MusicGen decodes without one)")
        return EncodecStreamDecoder(self, batch)

    def forward(self, x):
        """encodec.py:206-221 (inference part): returns the reconstruction trimmed to the input length and codes."""
        length = x.shape[-1]
        codes, scale = self.encode(x)
        out = self.decode(codes, scale)
        assert out.shape[-1] >= length, (out.shape[-1], length)
        return out[..., :length], codes

    @staticmethod
    def from_config_name(name: str, state_dict, device='cuda') -> 'EncodecModel':
        return EncodecModel(state_dict, ENCODEC_CONFIGS[name], device)


class _KernelLayers:
    """The layer operations of audiocraft_b200.streaming.DecoderStream on the decoder's kernels, each on a window that needs
    no padding."""

    def __init__(self, model: EncodecModel):
        self.m = model
        self.prec = model._dec_prec

    def conv(self, L, x):
        return self.m._conv(x.contiguous(), L, prec=self.prec, valid=True)

    def resblock(self, block, x, pad_left):
        shortcut, a, b = block
        m, x = self.m, x.contiguous()
        n = x.shape[-1] - (a['k'] - 1) * a['dilation']
        if shortcut is None and m._fused_block([a, b], 0, self.prec, x.shape[-1]):
            # the fused kernel writes every step of x; those whose window reaches into its zero padding are dropped
            return m._resblock(x, a, b, self.prec, pad_left=pad_left)[..., pad_left:pad_left + n]
        skip = x[..., pad_left:pad_left + n].contiguous()
        if shortcut is not None:
            skip = m._conv(skip, shortcut, prec=self.prec, valid=True)
        return m._conv(m._conv(x, a, prec=self.prec, valid=True), b, res=skip, prec=self.prec, valid=True)

    def convtr(self, L, x, trim_left, t_out):
        return self.m._convtr(x.contiguous(), L, prec=self.prec, window=(trim_left, t_out))

    def lstm_state(self, L, batch):
        z = lambda: torch.zeros((batch, L['dim']), device=self.m.device, dtype=torch.float32)   # noqa: E731
        return [(z(), z()) for _ in range(len(L['w_hh']))]

    def lstm(self, L, x, state):
        return self.m._lstm(x.contiguous(), L, prec=self.m._lstm_prec, state=state)

    def lstm_select(self, L, state, items):
        return [(h[items].contiguous(), c[items].contiguous()) for h, c in state]


class EncodecStreamDecoder:
    """`EncodecModel.stream_decoder(batch)`: the SEANet decoder with per-layer context (audiocraft_b200/streaming.py) on the
    kernels; the LSTM carries (h, c) between pushes."""

    def __init__(self, model: EncodecModel, batch: int):
        from .streaming import DecoderStream
        self.model, self.batch = model, batch
        self._stream = DecoderStream(model.dec, model.cfg, _KernelLayers(model), batch)

    @property
    def lookahead(self) -> int:
        """Latent frames past its own that a sample waits for once the stream is running."""
        return self._stream.lookahead

    def _out(self, y):
        if y is None:
            return torch.empty((self.batch, self.model.channels, 0), device=self.model.device, dtype=torch.float32)
        return y

    def select(self, items: tp.List[int]) -> 'EncodecStreamDecoder':
        """A stream decoder of the given items only, in this one's state (see streaming.DecoderStream.select)."""
        with torch.cuda.device(self.model.device):
            out = copy.copy(self)
            out.batch, out._stream = len(items), self._stream.select(list(items))
            return out

    def push(self, codes: torch.Tensor) -> torch.Tensor:
        assert codes.dim() == 3 and codes.shape[0] == self.batch, (tuple(codes.shape), self.batch)
        with torch.cuda.device(self.model.device):
            if codes.shape[-1] == 0:
                return self._out(None)
            return self._out(self._stream.push(self.model.decode_latent(codes)))

    def flush(self) -> torch.Tensor:
        with torch.cuda.device(self.model.device):
            return self._out(self._stream.flush())


class _StereoStreamDecoder:
    """The mono stream decoder over 2B items (left channels, then right), as `InterleaveStereoCompressionModel.decode`."""

    def __init__(self, wrapper: 'InterleaveStereoCompressionModel', inner, batch: int):
        self.wrapper, self.inner, self.batch = wrapper, inner, batch

    @property
    def lookahead(self) -> int:
        return self.inner.lookahead

    def _split(self, audio):
        return torch.cat([audio[:self.batch], audio[self.batch:]], dim=1)

    def select(self, items: tp.List[int]) -> '_StereoStreamDecoder':
        items = list(items)
        return _StereoStreamDecoder(self.wrapper, self.inner.select(items + [i + self.batch for i in items]), len(items))

    def push(self, codes: torch.Tensor) -> torch.Tensor:
        B, K, T = codes.shape
        assert B == self.batch and K == self.wrapper.num_codebooks, (tuple(codes.shape), self.batch)
        if T == 0:
            return self._split(self.inner.push(codes.new_empty((2 * B, K // 2, 0))))
        c0, c1 = self.wrapper.get_left_right_codes(codes)
        return self._split(self.inner.push(torch.cat([c0, c1], dim=0)))

    def flush(self) -> torch.Tensor:
        return self._split(self.inner.flush())


class InterleaveStereoCompressionModel(CompressionModel):
    """Stereo wrapper over a mono compression model: both channels share the codec and their codebooks are interleaved
    (`b (k c) t`, or per timestep `b k (t c)`).  Mirror of audiocraft/models/encodec.py:393-506 — same layouts, same
    properties; the two channels go through the kernels as ONE batch of 2B mono items (items are independent, so this
    equals the reference's two separate passes)."""

    def __init__(self, model: CompressionModel, per_timestep: bool = False):
        self.model = model
        self.per_timestep = per_timestep
        assert self.model.channels == 1, "Wrapped model is expected to be for monophonic audio"

    @property
    def total_codebooks(self):
        return self.model.total_codebooks

    @property
    def num_codebooks(self):
        """Active number of codebooks *after* interleaving (encodec.py:420-426)."""
        return self.model.num_codebooks if self.per_timestep else self.model.num_codebooks * 2

    def set_num_codebooks(self, n: int):
        """Sets the number of codebooks *before* interleaving (encodec.py:428-433)."""
        self.model.set_num_codebooks(n)

    @property
    def num_virtual_steps(self) -> float:
        return 2 if self.per_timestep else 1

    @property
    def frame_rate(self) -> float:
        return self.model.frame_rate * self.num_virtual_steps

    @property
    def sample_rate(self) -> int:
        return self.model.sample_rate

    @property
    def channels(self) -> int:
        return 2

    @property
    def cardinality(self):
        return self.model.cardinality

    def forward(self, x):
        raise NotImplementedError("Not supported, use encode and decode.")

    def encode(self, x):
        B, C, T = x.shape
        assert C == self.channels, f"Expecting stereo audio but audio num channels is {C}"
        mono = x.transpose(0, 1).reshape(2 * B, 1, T)                       # [c0 items..., c1 items...]
        indices, scales = self.model.encode(mono)
        indices = indices.view(2, B, indices.shape[1], indices.shape[2])    # c b k t
        out_scales = None
        if scales is not None:
            out_scales = torch.stack([scales[:B], scales[B:]], dim=1)
        if self.per_timestep:
            indices = indices.permute(1, 2, 3, 0).reshape(B, indices.shape[2], -1)          # b k (t c)
        else:
            indices = indices.permute(1, 2, 0, 3).reshape(B, -1, indices.shape[3])          # b (k c) t
        return indices.contiguous(), out_scales

    def get_left_right_codes(self, codes):
        B = codes.shape[0]
        if self.per_timestep:
            c = codes.view(B, codes.shape[1], -1, 2).permute(3, 0, 1, 2)
        else:
            c = codes.view(B, -1, 2, codes.shape[2]).permute(2, 0, 1, 3)
        return c[0].contiguous(), c[1].contiguous()

    def decode(self, codes, scale=None):
        B, K, T = codes.shape
        assert T % self.num_virtual_steps == 0, "Provided codes' number of timesteps does not match"
        assert K == self.num_codebooks, "Provided codes' number of codebooks does not match"
        scale_c0, scale_c1 = None, None
        if scale is not None:
            assert scale.size(0) == B and scale.size(1) == 2, f"Scale has unexpected shape: {scale.shape}"
            scale_c0 = scale[0, ...]   # as written in the reference (encodec.py:492-493)
            scale_c1 = scale[1, ...]
        c0, c1 = self.get_left_right_codes(codes)
        if scale is None:
            audio = self.model.decode(torch.cat([c0, c1], dim=0), None)
            return torch.cat([audio[:B], audio[B:]], dim=1)
        return torch.cat([self.model.decode(c0, scale_c0), self.model.decode(c1, scale_c1)], dim=1)

    def decode_latent(self, codes):
        raise NotImplementedError("Not supported by interleaved stereo wrapped models.")

    def stream_decoder(self, batch: int, scale=None):
        """The wrapped codec's stream decoder over 2B mono items; pieces are [B, 2, m]."""
        if self.per_timestep:
            raise NotImplementedError("streaming decode of per-timestep interleaved codes is not built")
        if not hasattr(self.model, 'stream_decoder'):
            raise NotImplementedError(f"{type(self.model).__name__} has no stream decoder")
        if scale is not None:
            raise NotImplementedError("streaming decode with a renormalisation scale is not built (MusicGen decodes without one)")
        return _StereoStreamDecoder(self, self.model.stream_decoder(2 * batch), batch)


def get_wrapped_compression_model(compression_model: CompressionModel, interleave_stereo_codebooks: tp.Optional[dict] = None,
                                  compression_model_n_q: tp.Optional[int] = None) -> CompressionModel:
    """audiocraft/models/builders.py:338-351 with the two cfg entries passed explicitly."""
    if interleave_stereo_codebooks and interleave_stereo_codebooks.get('use'):
        kwargs = {k: v for k, v in interleave_stereo_codebooks.items() if k != 'use'}
        compression_model = InterleaveStereoCompressionModel(compression_model, **kwargs)
    if compression_model_n_q is not None:
        compression_model.set_num_codebooks(compression_model_n_q)
    return compression_model


# ----------------------------------------------------------------------------- HuggingFace-format checkpoints

def hf_encodec_to_reference(hf_state_dict: tp.Dict[str, torch.Tensor], hf_config) -> tp.Tuple[dict, dict]:
    """Translate a `transformers.EncodecModel` checkpoint (what the reference loads for `facebook/encodec_*` through
    `HFEncodecCompressionModel`, audiocraft/models/encodec.py:119-121, 323-392) into the reference's own state_dict layout +
    hyper-parameters.  HF's implementation is the same algorithm with renamed modules
    (transformers/models/encodec/modeling_encodec.py), so the converted weights run on the kernels unchanged.
    norm_type 'time_group_norm' (the 48 kHz codec) maps `*.norm.{weight,bias}` to the reference's `...conv.norm.*` /
    `...convtr.norm.*`; its chunking (chunk_length_s / overlap) is carried in cfg as chunk_length / chunk_stride."""
    c = hf_config
    norm = getattr(c, 'norm_type', 'weight_norm')
    if norm not in ('weight_norm', 'time_group_norm'):
        raise NotImplementedError(f"HF EnCodec norm_type '{norm}' is not built (weight_norm, time_group_norm)")
    hop = int(math.prod(c.upsampling_ratios))
    frame_rate = math.ceil(c.sampling_rate / hop)
    n_qs = [int(bw * 1000 // (frame_rate * math.log2(c.codebook_size))) for bw in c.target_bandwidths]
    cfg = dict(channels=c.audio_channels, dimension=c.hidden_size, n_filters=c.num_filters,
               n_residual_layers=c.num_residual_layers, ratios=list(c.upsampling_ratios), kernel_size=c.kernel_size,
               last_kernel_size=c.last_kernel_size, residual_kernel_size=c.residual_kernel_size,
               dilation_base=c.dilation_growth_rate, causal=c.use_causal_conv, pad_mode=c.pad_mode, compress=c.compress,
               lstm=c.num_lstm_layers, norm=norm, trim_right_ratio=c.trim_right_ratio,
               sample_rate=c.sampling_rate, n_q=max(n_qs), bins=c.codebook_size, renormalize=c.normalize,
               true_skip=not c.use_conv_shortcut, possible_num_codebooks=n_qs,
               target_bandwidths=list(c.target_bandwidths), chunk_length=c.chunk_length, chunk_stride=c.chunk_stride)
    if norm == 'time_group_norm':
        cfg['norm_params'] = dict(eps=1e-5)   # nn.GroupNorm's default, which transformers' EncodecConv1d keeps
    plan = encodec_layers(cfg)
    kinds = {}
    for layer in plan['encoder'] + plan['decoder']:
        side, _, idx = layer['prefix'].split('.')[:3]
        kinds[(side, idx)] = layer['kind']
    sd = {}
    for k, v in hf_state_dict.items():
        parts = k.split('.')
        if parts[0] in ('encoder', 'decoder'):
            side, idx = parts[0], parts[2]
            rest = '.'.join(parts[3:])
            rest = rest.replace('parametrizations.weight.original0', 'weight_g').replace('parametrizations.weight.original1', 'weight_v')
            if rest.startswith('lstm.'):
                sd[f'{side}.model.{idx}.{rest}'] = v
                continue
            toks = rest.split('.')
            if toks[0] == 'block':               # block.<j>.{conv,norm}.<param> -> block.<j>.conv.{conv,norm}.<param>
                outer, mod, tail = f'block.{toks[1]}.conv', toks[2], toks[3:]
            elif toks[0] == 'shortcut':          # shortcut.{conv,norm}.<param> -> shortcut.conv.{conv,norm}.<param>
                outer, mod, tail = 'shortcut.conv', toks[1], toks[2:]
            else:                                # {conv,norm}.<param> -> {conv,convtr}.{conv,convtr,norm}.<param>
                outer = 'convtr' if kinds.get((side, idx)) == 'convtr' else 'conv'
                mod, tail = toks[0], toks[1:]
            inner = outer.split('.')[-1] if mod == 'conv' else 'norm'
            sd[f'{side}.model.{idx}.{outer}.{inner}.{".".join(tail)}'] = v
        elif parts[0] == 'quantizer':
            sd[f'quantizer.vq.layers.{parts[2]}._codebook.{parts[4]}'] = v
    return sd, cfg


def chunk_bounds(length: int, chunk_length: tp.Optional[int], chunk_stride: tp.Optional[int]) -> tp.List[tp.Tuple[int, int]]:
    """[start, end) of each chunk transformers' EncodecModel.encode cuts: offsets 0, stride, 2*stride, ... < length, each
    chunk_length long or cut by the end of the input; one chunk when the codec is not chunked."""
    if chunk_length is None:
        return [(0, length)]
    return [(o, min(o + chunk_length, length)) for o in range(0, length, chunk_stride)]


class _HFEncodecAPI:
    """`HFEncodecCompressionModel.model`: transformers' `EncodecModel.encode` / `.decode` (return_dict=False results), on the
    kernels.  This is what the reference's users call for audio longer than one chunk of a chunked codec."""

    def __init__(self, owner: 'HFEncodecCompressionModel', config):
        self._m = owner
        self.config = config

    def encode(self, input_values, padding_mask=None, bandwidth=None):
        """-> (audio_codes [n_chunks, B, K, frame_len], audio_scales: list of n_chunks [B, 1] (or None), last_frame_pad_length)."""
        return self._m._encode_chunks(input_values, padding_mask, bandwidth)

    def decode(self, audio_codes, audio_scales, padding_mask=None, last_frame_pad_length=0):
        """-> (audio_values [B, C, T],)."""
        return (self._m._decode_chunks(audio_codes, audio_scales, padding_mask, last_frame_pad_length),)


class HFEncodecCompressionModel(EncodecModel):
    """`facebook/encodec_*` checkpoints on the CUDA kernels: same surface as the reference's wrapper
    (audiocraft/models/encodec.py:323-392), incl. the restriction of `set_num_codebooks` to the bandwidths the
    checkpoint declares.  The 48 kHz codec cuts audio into 1 s chunks (stride 47 520) that are renormalised, encoded and
    decoded independently and joined by a linear overlap-add; all chunks of one length go through the kernels as one batch
    of items.  `.model.encode` / `.model.decode` take full-length audio, as transformers' model does."""

    def __init__(self, hf_state_dict, hf_config, device='cuda', **kw):
        sd, cfg = hf_encodec_to_reference(hf_state_dict, hf_config)
        super().__init__(sd, cfg, device, **kw)
        self.possible_num_codebooks = cfg['possible_num_codebooks']
        self.set_num_codebooks(max(self.possible_num_codebooks))
        self.model = _HFEncodecAPI(self, hf_config)

    @property
    def frame_rate(self):
        return self._frame_rate

    def set_num_codebooks(self, n: int):
        if n not in self.possible_num_codebooks:
            raise ValueError(f"Allowed values for num codebooks: {self.possible_num_codebooks}")
        self.n_q = n

    def _n_q_for_bandwidth(self, bandwidth):
        """EncodecResidualVectorQuantizer.get_num_quantizers_for_bandwidth, behind EncodecModel.encode's bandwidth check."""
        bws = self.cfg['target_bandwidths']
        if bandwidth is None:
            bandwidth = bws[0]
        if bandwidth not in bws:
            raise ValueError(f"This model doesn't support the bandwidth {bandwidth}. Select one of {bws}.")
        bw_per_q = math.log2(self.bins) * math.ceil(self.sample_rate / encodec_hop(self.cfg))
        return int(max(1, math.floor(bandwidth * 1000 / bw_per_q)))

    def _encode_chunks(self, x, padding_mask=None, bandwidth=None):
        n_q = self._n_q_for_bandwidth(bandwidth)
        with torch.cuda.device(self.device):
            x = self._in(x)
            if padding_mask is not None:
                x = x * padding_mask.to(self.device).view(x.shape[0], -1, x.shape[-1]).bool()
            bounds = chunk_bounds(x.shape[-1], self.cfg['chunk_length'], self.cfg['chunk_stride'])
            codes, scales = [None] * len(bounds), [None] * len(bounds)
            for length in sorted({e - s for s, e in bounds}, reverse=True):   # one batch of items per chunk length
                idx = [i for i, (s, e) in enumerate(bounds) if e - s == length]
                batch = torch.cat([x[..., bounds[i][0]:bounds[i][1]] for i in idx]).contiguous()   # [chunk][item]
                batch, scale = self.preprocess(batch)
                c = self.quantize(self._run(batch.contiguous(), self.enc, self._enc_prec), n_q)
                for j, i in enumerate(idx):
                    codes[i] = c[j * x.shape[0]:(j + 1) * x.shape[0]]
                    scales[i] = None if scale is None else scale[j * x.shape[0]:(j + 1) * x.shape[0]]
            frames = codes[0].shape[-1]
            if any(c.shape[-1] != frames for c in codes[:-1]):
                raise ValueError(f"input length {x.shape[-1]} gives chunks of {[c.shape[-1] for c in codes]} frames: every chunk "
                                 "but the last must have as many frames as the first")
            pad = frames - codes[-1].shape[-1]
            if pad > 0:
                codes[-1] = torch.nn.functional.pad(codes[-1], (0, pad), value=0)
            return torch.stack(codes), scales, pad

    def _decode_chunks(self, audio_codes, audio_scales, padding_mask=None, last_frame_pad_length=0):
        n = len(audio_codes)
        if self.cfg['chunk_length'] is None and n != 1:
            raise ValueError(f"Expected one frame, got {n}")
        pad = last_frame_pad_length or 0
        with torch.cuda.device(self.device):
            codes = audio_codes.to(self.device, torch.int64)
            scales = [audio_scales[i] for i in range(n)]
            last = self._run(self.decode_latent(codes[-1][..., :codes.shape[-1] - pad]), self.dec, self._dec_prec)
            B = last.shape[0]
            if self.cfg['chunk_length'] is None:
                out = last if scales[0] is None else last * scales[0].to(self.device).view(-1, 1, 1)
            else:
                full = None
                if n > 1:
                    full = self._run(self.decode_latent(codes[:-1].reshape(-1, *codes.shape[2:])), self.dec, self._dec_prec)
                sc = None
                if scales[0] is not None:
                    sc = torch.stack([s.to(self.device, torch.float32).reshape(-1).expand(B) for s in scales]).contiguous()
                t_frame = full.shape[-1] if full is not None else last.shape[-1]
                stride = self.cfg['chunk_stride']
                t_total = stride * (n - 1) + last.shape[-1]
                out = torch.empty((B, last.shape[1], t_total), device=self.device, dtype=torch.float32)
                _lib.check(self._lib.acb_overlap_add(_lib.ptr(full), _lib.ptr(last), _lib.ptr(sc), _lib.ptr(out), n, B,
                                                     last.shape[1], t_frame, last.shape[-1], stride, t_total, _lib.stream()),
                           'overlap_add')
                self.launches += 1
            if padding_mask is not None and padding_mask.shape[-1] < out.shape[-1]:
                out = out[..., :padding_mask.shape[-1]]
            return out

    def encode(self, x):
        """encodec.py:347-353: one chunk only; longer input goes through `.model.encode`."""
        bandwidth = self.cfg['target_bandwidths'][self.possible_num_codebooks.index(self.num_codebooks)]
        n = len(chunk_bounds(x.shape[-1], self.cfg['chunk_length'], self.cfg['chunk_stride']))
        assert n == 1, (f"input of {x.shape[-1]} samples spans {n} chunks of {self.cfg['chunk_length']}: the reference wrapper "
                        "encodes one chunk (`assert len(res[0]) == 1`); use `.model.encode` / `.model.decode` for longer audio")
        codes, scales, _ = self.model.encode(x, None, bandwidth)
        return codes[0], scales[0]

    def stream_decoder(self, batch: int, scale=None):
        raise NotImplementedError("streaming decode of a transformers EnCodec checkpoint is not built: its chunking is an "
                                  "overlap-add of independently decoded chunks")

    def decode(self, codes, scale=None):
        """encodec.py:355-361: `self.model.decode(codes[None], scale)`.  The reference passes the [B, 1] scale where transformers
        expects one [B, 1] scale per chunk, so chunk 0 takes row 0: item 0's scale is applied to EVERY item (kept as written)."""
        return self.model.decode(codes[None], [None] if scale is None else scale)[0]

    @staticmethod
    def from_pretrained_dir(path: str, device='cuda'):
        """A local snapshot of an HF EnCodec repo (config.json + weights); the hub itself is unreachable offline."""
        from transformers import EncodecModel as _HF
        m = _HF.from_pretrained(path, local_files_only=True)
        return HFEncodecCompressionModel(m.state_dict(), m.config, device)
