"""MusicGen LM on H100: host-side mirror of ``audiocraft.models.lm.LMModel`` over the C-ABI decode kernels.

Keeps ``LMModel.generate``'s signature and semantics (audiocraft/models/lm.py:420-587) and the attributes its callers
read (``condition_provider, fuser, card, n_q, num_codebooks, special_token_id, cfg_coef``), but the hot loop
(lm.py:540-565: ~1500 Python iterations x ~15 kernels x L layers in the reference) runs as one CUDA-graph launch per
step with sampling, CFG mixing, masking and the sequence write-back on the device.

Weights: reference-layout LM ``state_dict`` (SURVEY.md section 8b), cast to fp16 like the reference does on CUDA
(audiocraft/models/loaders.py:115-118); LayerNorm parameters stay fp32.  Accumulation, residual stream, LayerNorm and
softmax are fp32.  No CPU path exists.
"""
import typing as tp
from dataclasses import dataclass

import torch

from . import _lib
from .conditioners import (ConditionFuser, ConditioningAttributes, ConditioningProvider, nullify_all)
from .patterns import DelayedPatternProvider

import ctypes as C


@dataclass
class LMOutput:
    """audiocraft/models/lm.py:95-101: logits [B,K,T,card] (NaN where the pattern gives no prediction) and mask [B,K,T]."""
    logits: torch.Tensor
    mask: torch.Tensor


class LMModel:
    def __init__(self, state_dict: tp.Dict[str, torch.Tensor], cfg: dict,
                 condition_provider: tp.Optional[ConditioningProvider] = None,
                 fuser: tp.Optional[ConditionFuser] = None, device='cuda'):
        self.device = _lib.require_cuda(device)
        self._lib = _lib.lib()
        self.cfg_dict = dict(cfg)
        self.dim, self.num_heads, self.num_layers = cfg['dim'], cfg['num_heads'], cfg['num_layers']
        self.card, self.n_q = cfg['card'], cfg['n_q']
        self.ffn_dim = int(cfg['hidden_scale'] * cfg['dim'])
        self.cfg_coef = cfg.get('cfg_coef', 3.0)
        self.two_step_cfg = cfg.get('two_step_cfg', False)
        self.cross_attention = bool(cfg.get('cross_attention', True))
        self.pattern_provider = DelayedPatternProvider(self.n_q, delays=cfg['delays'])
        self.condition_provider = condition_provider
        self.fuser = fuser if fuser is not None else ConditionFuser({'cross': ['description']})
        # `prepend` fuser (MusicGen-melody): the conditions run as a prefix of the sequence, prefilled into the KV cache
        self.has_prefix = bool(self.fuser.fuse2cond.get('prepend'))
        if self.condition_provider is not None:
            self.condition_provider.to(self.device)
            cp = {k[len('condition_provider.'):]: v for k, v in state_dict.items() if k.startswith('condition_provider.')}
            if cp:
                self.condition_provider.load_state_dict({k: v.float() for k, v in cp.items()}, strict=False)
        assert self.dim == self.num_heads * 64, "the decode kernels are built for head_dim 64 (all MusicGen scales)"
        self._handle = None
        self._bufs = None
        self._shape = None
        self._debug_noise_fn = None
        self.launches_per_step = 0
        with torch.cuda.device(self.device):
            self._load_weights(state_dict, cfg)

    # ------------------------------------------------------------------ weights
    def _load_weights(self, sd, cfg):
        dev, L, d = self.device, self.num_layers, self.dim

        def h(t):
            return t.to(dev, torch.float16).contiguous()

        def stack(fmt, rows=None):
            first = sd[fmt.format(0)]
            shape = first.shape if rows is None else (rows[1] - rows[0],) + tuple(first.shape[1:])
            out = torch.empty((L,) + tuple(shape), device=dev, dtype=torch.float16)
            for li in range(L):
                t = sd[fmt.format(li)]
                out[li].copy_(t if rows is None else t[rows[0]:rows[1]])
            return out

        w = {}
        w['emb'] = torch.stack([h(sd[f'emb.{k}.weight']) for k in range(self.n_q)]).contiguous()
        half = d // 2
        adim = torch.arange(half, dtype=torch.float32)
        # divisor table of create_sin_embedding (transformer.py:84-88), computed by the same torch ops
        w['inv_freq'] = (torch.tensor(float(cfg['max_period'])) ** (adim / (half - 1))).to(dev).contiguous()
        p = 'transformer.layers.{}.'
        w['w_qkv'] = stack(p + 'self_attn.in_proj_weight')
        w['w_o'] = stack(p + 'self_attn.out_proj.weight')
        if self.cross_attention:
            w['w_cq'] = stack(p + 'cross_attention.in_proj_weight', rows=(0, d))
            w['w_ckv'] = stack(p + 'cross_attention.in_proj_weight', rows=(d, 3 * d))
            w['w_co'] = stack(p + 'cross_attention.out_proj.weight')
        else:
            w['w_cq'] = w['w_ckv'] = w['w_co'] = None
        w['w_ff1'] = stack(p + 'linear1.weight')
        w['w_ff2'] = stack(p + 'linear2.weight')
        ln = torch.zeros((L, 6, d), device=dev, dtype=torch.float32)
        for li in range(L):
            names = ['norm1', 'norm_cross', 'norm2'] if self.cross_attention else ['norm1', None, 'norm2']
            for j, n in enumerate(names):
                if n is None:
                    continue
                ln[li, 2 * j] = sd[f'transformer.layers.{li}.{n}.weight'].float()
                ln[li, 2 * j + 1] = sd[f'transformer.layers.{li}.{n}.bias'].float()
        w['ln'] = ln
        w['out_norm'] = torch.stack([sd['out_norm.weight'].float(), sd['out_norm.bias'].float()]).to(dev).contiguous()
        w['heads'] = torch.cat([h(sd[f'linears.{k}.weight']) for k in range(self.n_q)], dim=0).contiguous()
        # positional_embedding (transformer.py:632-637): rotary frequencies computed by the same torch ops as rope.py:68-69
        self.positional_embedding = cfg.get('positional_embedding', 'sin')
        assert self.positional_embedding in ('sin', 'rope', 'sin_rope')
        if self.positional_embedding != 'sin':
            adim2 = torch.arange(0, 64, 2, dtype=torch.float32)[:32]
            w['rope_freq'] = (1.0 / (float(cfg['max_period']) ** (adim2 / 64))).to(dev).contiguous()
        else:
            w['rope_freq'] = None
        self._w = w
        self.weight_bytes_per_step = sum(
            t.numel() * t.element_size() for k, t in w.items()
            if t is not None and k not in ('emb', 'inv_freq', 'w_ckv', 'rope_freq'))

    # ------------------------------------------------------------------ reference attributes
    @property
    def special_token_id(self) -> int:
        return self.card

    @property
    def num_codebooks(self) -> int:
        return self.n_q

    def parameters(self):
        return iter([t for t in self._w.values() if t is not None])

    def eval(self):
        return self

    def _config(self, max_rows: int = 1, max_seq: int = 2, max_text: int = 1) -> _lib.LMConfig:
        return _lib.LMConfig(self.dim, self.num_heads, self.num_layers, self.ffn_dim, self.n_q, self.card,
                             int(self.cross_attention), max_rows, max_seq, max_text,
                             float(self.cfg_dict.get('positional_scale', 1.0)),
                             {'sin': 0, 'rope': 1, 'sin_rope': 2}[self.positional_embedding])

    def _weights(self) -> _lib.LMWeights:
        return _lib.LMWeights(*[_lib.ptr(self._w[n]) for n in ('emb', 'inv_freq', 'w_qkv', 'w_o', 'w_cq', 'w_ckv',
                                                              'w_co', 'w_ff1', 'w_ff2', 'ln', 'out_norm', 'heads', 'rope_freq')])

    # ------------------------------------------------------------------ device state
    def _ensure(self, rows: int, seq_len: int, text_len: int, batch: int):
        shape = self._shape
        if shape is not None and rows <= shape[0] and seq_len <= shape[1] and text_len <= shape[2] and batch <= shape[3]:
            return
        self._destroy()
        dev, d, H, L = self.device, self.dim, self.num_heads, self.num_layers
        max_rows = rows if shape is None else max(rows, shape[0])
        max_seq = seq_len if shape is None else max(seq_len, shape[1])
        max_text = max(1, text_len if shape is None else max(text_len, shape[2]))
        max_batch = batch if shape is None else max(batch, shape[3])
        # activation buffers also hold the (token, row) pairs of a prompt-prefill pass (acb_lm_prefill): up to
        # ACB_LM_PREFILL_ROWS, or one position of every row above that
        rp = self._lib.acb_lm_rows_pad(max_rows)
        if rp < 0:
            _lib.check(rp, 'lm_rows_pad')
        rp = max(rp, _lib.ACB_LM_PREFILL_ROWS)
        f16, f32 = torch.float16, torch.float32
        b = {}
        b['x'] = torch.zeros((rp, d), device=dev, dtype=f32)
        b['h16'] = torch.zeros((rp, d), device=dev, dtype=f16)
        b['a16'] = torch.zeros((rp, d), device=dev, dtype=f16)
        b['f16'] = torch.zeros((rp, self.ffn_dim), device=dev, dtype=f16)
        b['q32'] = torch.zeros((rp, d), device=dev, dtype=f32)
        b['part'] = torch.zeros((_lib.ACB_LM_PART_SLOTS, rp, max(3 * d, self.ffn_dim, self.n_q * self.card)), device=dev, dtype=f32)
        b['logits'] = torch.zeros((rp, self.n_q * self.card), device=dev, dtype=f32)
        b['k_cache'] = torch.zeros((L, max_rows, H, max_seq, 64), device=dev, dtype=f16)
        b['v_cache'] = torch.zeros((L, max_rows, H, max_seq, 64), device=dev, dtype=f16)
        if self.cross_attention:
            b['ck_cache'] = torch.zeros((L, max_rows, H, max_text, 64), device=dev, dtype=f16)
            b['cv_cache'] = torch.zeros((L, max_rows, H, max_text, 64), device=dev, dtype=f16)
            mp = (max_rows * max_text + 63) // 64 * 64
            b['cross16'] = torch.zeros((mp, d), device=dev, dtype=f16)
        else:
            b['ck_cache'] = b['cv_cache'] = b['cross16'] = None
        b['seq'] = torch.full((max_batch, self.n_q, max_seq), -1, device=dev, dtype=torch.int64)
        b['seq_mask'] = torch.zeros((self.n_q, max_seq), device=dev, dtype=torch.uint8)
        b['pos'] = torch.zeros(4, device=dev, dtype=torch.int32)
        b['noise'] = torch.ones((max_batch, self.n_q, self.card), device=dev, dtype=f32)
        self._bufs = b
        cfg = self._config(max_rows, max_seq, max_text)
        wts = self._weights()
        bufs = _lib.LMBuffers(*[_lib.ptr(b[n]) for n in ('x', 'h16', 'a16', 'f16', 'q32', 'part', 'logits', 'k_cache',
                                                         'v_cache', 'ck_cache', 'cv_cache', 'cross16', 'seq',
                                                         'seq_mask', 'pos', 'noise')])
        handle = C.c_void_p()
        _lib.check(self._lib.acb_lm_create(C.byref(cfg), C.byref(wts), C.byref(bufs), C.byref(handle)), 'lm_create')
        self._handle = handle
        self._shape = (max_rows, max_seq, max_text, max_batch)

    def _destroy(self):
        if self._handle is not None:
            torch.cuda.synchronize(self.device)
            self._lib.acb_lm_destroy(self._handle)
            self._handle = None
            self._bufs = None

    def __del__(self):
        try:
            self._destroy()
        except Exception:
            pass

    # ------------------------------------------------------------------ conditions (lm.py:488-511)
    def _prepare_conditions(self, conditions, two_step_cfg, cfg_coef_beta):
        return self._condition_tensors(conditions, cfg_coef_beta)[0]

    def _condition_tensors(self, conditions, cfg_coef_beta=None):
        """(cross_attention_src, prefix) of [conditions; null conditions], each None when the fuser produces none."""
        if not conditions:
            return None, None
        assert self.condition_provider is not None, "conditions given but the model has no condition_provider"
        if cfg_coef_beta is not None:
            # lm.py:490-496: [conditions; conditions without their description; null conditions].  The style-only rows need
            # a 'self_wav' conditioner (conditioners.py:231-234 asserts the same); it is a front-end outside the hot path,
            # so double CFG is reachable with a pre-computed 3B-row `cross_attention_src`.
            for c in conditions:
                assert 'description' in c.text and 'self_wav' in getattr(c, 'wav', {}), \
                    "double CFG needs 'description' and 'self_wav' conditions (conditioners.py:231-234)"
            raise NotImplementedError("style (self_wav) conditioner front-end is not built; pass cross_attention_src with "
                                      "[cond; style-only; null] rows")
        null_conditions = nullify_all(conditions)
        tokenized = self.condition_provider.tokenize(list(conditions) + null_conditions)
        tensors = self.condition_provider(tokenized)
        return self.fuser.cross_source(tensors), self.fuser.prefix_source(tensors)

    def _check_prefix(self, prefix, rows, two_step_cfg=False, cfg_coef_beta=None):
        """The condition prefix as the contiguous fp32 CUDA tensor [rows, P, d] acb_lm_begin_prefix takes (None: P = 0)."""
        if prefix is None:
            return None, 0
        if two_step_cfg:
            raise NotImplementedError("two_step_cfg with a condition prefix (prepend fuser) is not built")
        if cfg_coef_beta is not None:
            raise NotImplementedError("double CFG (cfg_coef_beta) with a condition prefix (prepend fuser) is not built")
        prefix = prefix.to(self.device, torch.float32).contiguous()
        assert prefix.dim() == 3 and prefix.shape[2] == self.dim and prefix.shape[0] == rows, \
            f"prefix must be [rows={rows}, P, {self.dim}], got {tuple(prefix.shape)}"
        if prefix.shape[1] == 0:
            return None, 0
        return prefix, prefix.shape[1]

    def _begin(self, cross, prefix, P, B, rows, text_len, S, samp):
        _lib.check(self._lib.acb_lm_begin_prefix(self._handle, _lib.ptr(cross), _lib.ptr(prefix), P, B, rows, text_len, S,
                                                 C.byref(samp), _lib.stream()), 'lm_begin')

    # ------------------------------------------------------------------ generation
    @torch.no_grad()
    def generate(self, prompt: tp.Optional[torch.Tensor] = None,
                 conditions: tp.List[ConditioningAttributes] = [],
                 num_samples: tp.Optional[int] = None, max_gen_len: int = 256, use_sampling: bool = True,
                 temp: float = 1.0, top_k: int = 250, top_p: float = 0.0, cfg_coef: tp.Optional[float] = None,
                 cfg_coef_beta: tp.Optional[float] = None, two_step_cfg: tp.Optional[bool] = None,
                 remove_prompts: bool = False, check: bool = False,
                 callback: tp.Optional[tp.Callable[[int, int], None]] = None,
                 cross_attention_src: tp.Optional[torch.Tensor] = None,
                 prefix: tp.Optional[torch.Tensor] = None) -> torch.Tensor:
        """Same contract as LMModel.generate (lm.py:420-587).  ``cross_attention_src`` is an extension: a pre-computed
        [2B,T,d] (or [B,T,d] without CFG) condition tensor, bypassing the host conditioners.  ``prefix`` likewise: a
        pre-computed [rows,P,d] condition prefix (the `prepend` fuser's output, one per row) for a model that has one."""
        if num_samples is None:
            if prompt is not None:
                num_samples = prompt.shape[0]
            elif conditions:
                num_samples = len(conditions)
            elif cross_attention_src is not None:
                raise ValueError("num_samples is required with cross_attention_src")
            else:
                num_samples = 1
        two_step_cfg = self.two_step_cfg if two_step_cfg is None else two_step_cfg
        if self.has_prefix and two_step_cfg:
            raise NotImplementedError("two_step_cfg with a condition prefix (prepend fuser) is not built")
        if self.has_prefix and cfg_coef_beta is not None:
            raise NotImplementedError("double CFG (cfg_coef_beta) with a condition prefix (prepend fuser) is not built")
        if cross_attention_src is not None or prefix is not None:
            cross = cross_attention_src
        else:
            cross, prefix = self._condition_tensors(conditions, cfg_coef_beta)
        B, K = num_samples, self.n_q
        # lm.py:387 quirk: the two-step branch uses self.cfg_coef, not the argument.  (With exact-zero null rows the
        # two passes are numerically the batched pass: V = 0 makes the null branch independent of its padding.)
        coef = self.cfg_coef if (cfg_coef is None or (two_step_cfg and cross is not None)) else cfg_coef
        with torch.cuda.device(self.device):
            if prompt is None:
                assert num_samples > 0
                prompt = torch.zeros((B, K, 0), dtype=torch.long, device=self.device)
            prompt = prompt.to(self.device, torch.long)
            assert prompt.shape[:2] == (B, K), "Inconsistent inputs shapes"
            T0 = prompt.shape[-1]
            start_offset = T0
            assert start_offset < max_gen_len

            pattern = self.pattern_provider.get_pattern(max_gen_len)
            unknown_token = -1
            gen_codes = torch.full((B, K, max_gen_len), unknown_token, dtype=torch.long, device=self.device)
            gen_codes[..., :start_offset] = prompt
            gen_sequence, _, mask = pattern.build_pattern_sequence(gen_codes, self.special_token_id)
            start_offset_sequence = pattern.get_first_step_with_timesteps(start_offset)
            assert start_offset_sequence is not None
            S = gen_sequence.shape[-1]

            rows = B
            text_len = 0
            if cross is not None:
                cross = cross.to(self.device, torch.float32).contiguous()
                assert cross.dim() == 3 and cross.shape[2] == self.dim
                assert cross.shape[0] in (B, 2 * B, 3 * B), \
                    "condition rows must be B (no CFG), 2B ([cond; null]) or 3B ([cond; style-only; null], double CFG)"
                assert (cross.shape[0] == 3 * B) == (cfg_coef_beta is not None), \
                    "cfg_coef_beta goes with 3B condition rows (lm.py:362-376)"
                rows, text_len = cross.shape[0], cross.shape[1]
            elif prefix is not None:
                rows = prefix.shape[0]
                assert rows in (B, 2 * B), "prefix rows must be B (no CFG) or 2B ([cond; null])"
            prefix, P = self._check_prefix(prefix, rows, two_step_cfg, cfg_coef_beta)
            self._ensure(rows, P + S, text_len, B)
            bufs = self._bufs
            bufs['seq'][:B, :, :S] = gen_sequence
            bufs['seq_mask'][:, :S] = mask.to(torch.uint8)
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
            samp = _lib.LMSampling(int(bool(use_sampling)), float(temp), int(top_k), float(top_p), float(coef), seed,
                                   1 if self._debug_noise_fn is not None else 0,
                                   float(cfg_coef_beta) if cfg_coef_beta is not None else 0.0)
            self._begin(cross, prefix, P, B, rows, text_len, S, samp)
            self.launches_per_step = self._lib.acb_lm_launches_per_step(self._handle)
            n_steps = S - 1
            # Prompt prefill (the reference's multi-token first call, lm.py:513-534, transformer.py:240-247): positions
            # [0, start - 1) only feed the KV cache -- their tokens are known and the first sampled position is `start` -- so
            # they go through acb_lm_prefill, several positions per pass, instead of one decode step each.
            first = 0
            import os as _os
            if start_offset_sequence - 1 >= 2 and _os.environ.get('ACB_LM_PREFILL', '1') != '0':
                first = start_offset_sequence - 1
                _lib.check(self._lib.acb_lm_prefill(self._handle, 0, first, _lib.stream()), 'lm_prefill')
            if callback is None and self._debug_noise_fn is None:
                _lib.check(self._lib.acb_lm_steps(self._handle, n_steps - first, _lib.stream()), 'lm_steps')
            else:
                for pos in range(first, n_steps):
                    offset = pos + 1
                    if self._debug_noise_fn is not None:
                        bufs['noise'][:B].copy_(self._debug_noise_fn(offset, (B, K, self.card)).reshape(B, K, self.card))
                    _lib.check(self._lib.acb_lm_steps(self._handle, 1, _lib.stream()), 'lm_steps')
                    if callback is not None and offset >= start_offset_sequence:
                        callback(1 + offset - start_offset_sequence, S - start_offset_sequence)
            gen_sequence = bufs['seq'][:B, :, :S].clone()

            # lm.py:568-586
            assert not (gen_sequence == unknown_token).any()
            assert (gen_sequence == torch.where(mask[None, ...].expand(B, -1, -1), gen_sequence,
                                                self.special_token_id)).all()
            out_codes, _, out_mask = pattern.revert_pattern_sequence(gen_sequence, special_token=unknown_token)
            assert (out_codes[..., :max_gen_len] != unknown_token).all()
            assert (out_mask[..., :max_gen_len] == 1).all()
            out_start_offset = start_offset if remove_prompts else 0
            out_codes = out_codes[..., out_start_offset:max_gen_len]
            assert (out_codes >= 0).all() and (out_codes <= self.card).all()
            self.last_sequence = gen_sequence
            return out_codes

    # ------------------------------------------------------------------ streaming-state surface (modules/streaming.py:59-119)
    # The reference keeps `past_keys` / `past_values` ([rows, H, t, 64], transformer.py:266-298) per attention module and
    # `offsets` per transformer, reachable through StreamingModule.get/set_streaming_state; LMModel._sample_next_token uses
    # them to run two_step_cfg (lm.py:376-391).  Here the same observable state lives in the device KV cache + the device
    # position counter; the methods below expose it under the reference's key names.
    def streaming_begin(self, batch: int, cross: tp.Optional[torch.Tensor], max_len: int, cfg_coef: tp.Optional[float] = None,
                        cfg_coef_beta: tp.Optional[float] = None, prefix: tp.Optional[torch.Tensor] = None, **sampling):
        """Enter streaming mode for `batch` items (what `with lm.streaming():` + the first forward do in the reference):
        allocates / resets the caches, precomputes the cross-attention K/V of `cross` ([rows,T,d] rows = batch, 2*batch or
        3*batch), prefills the condition `prefix` ([rows,P,d], the first call's prepended conditions) and captures the step
        graph.  Then `streaming_step(tokens)` consumes one [B,K] column per call; offsets count the prefix, as the
        reference's transformer offsets do."""
        with torch.cuda.device(self.device):
            rows, text_len = batch, 0
            if cross is not None:
                cross = cross.to(self.device, torch.float32).contiguous()
                rows, text_len = cross.shape[0], cross.shape[1]
            elif prefix is not None:
                rows = prefix.shape[0]
            prefix, P = self._check_prefix(prefix, rows, False, cfg_coef_beta)
            self._ensure(rows, P + max_len + 1, text_len, batch)
            b = self._bufs
            b['seq'][:batch].fill_(-1)
            b['seq_mask'].fill_(1)
            samp = _lib.LMSampling(int(bool(sampling.get('use_sampling', False))), float(sampling.get('temp', 1.0)),
                                   int(sampling.get('top_k', 0)), float(sampling.get('top_p', 0.0)),
                                   float(self.cfg_coef if cfg_coef is None else cfg_coef), int(sampling.get('seed', 0)), 0,
                                   float(cfg_coef_beta) if cfg_coef_beta is not None else 0.0)
            self._begin(cross, prefix, P, batch, rows, text_len, max_len + 1, samp)
            self._stream = dict(batch=batch, rows=rows, max_len=max_len, prefix_len=P)

    @torch.no_grad()
    def streaming_step(self, tokens: torch.Tensor) -> torch.Tensor:
        """LMModel.forward on ONE column in streaming mode (lm.py:221-268 with S = 1): tokens [B,K] -> CFG-mixed logits
        [B,K,card]; the KV cache grows by one position."""
        st = self._stream
        with torch.cuda.device(self.device):
            pos = int(self._bufs['pos'][0].item()) - st['prefix_len']   # sequence column
            assert pos < st['max_len'], "streaming_begin(max_len) exceeded"
            self._bufs['seq'][:st['batch'], :, pos] = tokens.to(self.device, torch.long)
            self._bufs['seq'][:st['batch'], :, pos + 1] = -1
            out = torch.empty((st['batch'], self.n_q, self.card), device=self.device, dtype=torch.float32)
            _lib.check(self._lib.acb_lm_step_logits(self._handle, out.data_ptr(), _lib.stream()), 'lm_step_logits')
            return out

    def get_streaming_state(self) -> tp.Dict[str, torch.Tensor]:
        """StreamingModule.get_streaming_state (streaming.py:72-84) under the reference's key names: a COPY of the cached
        keys / values of every layer up to the current offset and the per-row offsets."""
        st, b = self._stream, self._bufs
        pos = int(b['pos'][0].item())
        rows = st['rows']
        state = {'transformer.offsets': torch.full((rows,), pos, dtype=torch.long, device=self.device)}
        for li in range(self.num_layers):
            state[f'transformer.layers.{li}.self_attn.past_keys'] = b['k_cache'][li, :rows, :, :pos].clone()
            state[f'transformer.layers.{li}.self_attn.past_values'] = b['v_cache'][li, :rows, :, :pos].clone()
        return state

    def set_streaming_state(self, state: tp.Dict[str, torch.Tensor]):
        """StreamingModule.set_streaming_state (streaming.py:86-103): restore offsets and cached keys / values."""
        st, b = self._stream, self._bufs
        rows = st['rows']
        offs = state['transformer.offsets']
        assert bool((offs == offs[0]).all()), "rows of one generate() share their offset"
        pos = int(offs[0].item())
        state = dict(state)
        state.pop('transformer.offsets')
        for li in range(self.num_layers):
            k = state.pop(f'transformer.layers.{li}.self_attn.past_keys')
            v = state.pop(f'transformer.layers.{li}.self_attn.past_values')
            assert k.shape == (rows, self.num_heads, pos, 64) and v.shape == k.shape, (k.shape, pos)
            b['k_cache'][li, :rows, :, :pos] = k
            b['v_cache'][li, :rows, :, :pos] = v
        assert len(state) == 0, list(state.keys())
        assert pos >= st['prefix_len'], "the state must include the condition prefix"
        b['pos'][0] = pos

    def reset_streaming(self):
        """StreamingModule.reset_streaming (streaming.py:64-70): forget the cached positions.  A condition prefix stays
        cached: the reference prepends it again on the first call after a reset, which is the same cache content."""
        self._bufs['pos'][0] = self._stream.get('prefix_len', 0) if getattr(self, '_stream', None) else 0

    @torch.no_grad()
    def teacher_forced_logits(self, sequence: torch.Tensor, cross: tp.Optional[torch.Tensor], cfg_coef: float,
                              n_steps: tp.Optional[int] = None, keep: tp.Optional[tp.Sequence[int]] = None,
                              raw: bool = False, prefix: tp.Optional[torch.Tensor] = None):
        """Feed a fully known delay-pattern sequence [B,K,S] token by token and return the (CFG-mixed when cross has
        2B rows) next-token logits [n_steps,B,K,card] -- LMModel.forward in streaming mode (lm.py:221-268), the
        quantity the parity tests compare against the oracle.  ``keep``: only these step indices are returned (in that
        order; every step still runs).  ``raw``: also return the un-mixed per-row logits [n,rows,K,card] ([cond; null]).
        ``prefix``: [rows,P,d] condition prefix prefilled in front of the sequence (its logits are not returned)."""
        with torch.cuda.device(self.device):
            sequence = sequence.to(self.device, torch.long)
            B, K, S = sequence.shape
            rows, text_len = B, 0
            if cross is not None:
                cross = cross.to(self.device, torch.float32).contiguous()
                rows, text_len = cross.shape[0], cross.shape[1]
            elif prefix is not None:
                rows = prefix.shape[0]
            prefix, P = self._check_prefix(prefix, rows)
            self._ensure(rows, P + S, text_len, B)
            bufs = self._bufs
            bufs['seq'][:B, :, :S] = sequence
            bufs['seq_mask'][:, :S] = 1
            samp = _lib.LMSampling(0, 1.0, 0, 0.0, float(cfg_coef), 0, 0)
            self._begin(cross, prefix, P, B, rows, text_len, S, samp)
            self.launches_per_step = self._lib.acb_lm_launches_per_step(self._handle)
            n = S - 1 if n_steps is None else n_steps
            slot = {i: j for j, i in enumerate(range(n) if keep is None else keep)}
            out = torch.empty((len(slot), B, K, self.card), device=self.device, dtype=torch.float32)
            raw_out = torch.empty((len(slot), rows, K, self.card), device=self.device, dtype=torch.float32) if raw else None
            last = max(slot) if slot else -1
            for i in range(min(n, last + 1)):
                j = slot.get(i)
                _lib.check(self._lib.acb_lm_step_logits(self._handle, out[j].data_ptr() if j is not None else None,
                                                        _lib.stream()), 'lm_step_logits')
                if raw and j is not None:
                    raw_out[j].copy_(bufs['logits'][:rows].view(rows, K, self.card))
            return (out, raw_out) if raw else out

    # ------------------------------------------------------------------ full-sequence forward (scoring)
    @torch.no_grad()
    def forward(self, sequence: torch.Tensor, conditions: tp.List[ConditioningAttributes] = [],
                condition_tensors: tp.Optional[tp.Dict[str, tp.Any]] = None, stage: int = -1, *,
                cross_attention_src: tp.Optional[torch.Tensor] = None,
                prefix: tp.Optional[torch.Tensor] = None) -> torch.Tensor:
        """LMModel.forward (lm.py:221-268): sequence [B,K,S] (codes or the special token `card`) -> logits [B,K,S,card], one
        causal pass over every position on the acb_lm_forward kernels.  The logits are fp32 (the reference returns fp16
        under CUDA autocast).  Conditions go through condition_provider and fuser without CFG rows, as in the reference;
        ``cross_attention_src`` [B,T_text,d] and ``prefix`` [B,P,d] are pre-computed condition tensors, as for generate.
        With a `prepend` fuser the prefix runs as the first P positions and its logits are dropped.  The decode state
        (KV caches, position, captured step) is neither read nor changed."""
        if stage >= 0:
            raise NotImplementedError("stage >= 0 (MAGNeT's per-stage attention masks) is not built")
        B, K, S = sequence.shape
        assert K == self.num_codebooks, "Sequence shape must match the specified number of codebooks"
        cross = cross_attention_src
        if cross is not None or prefix is not None:
            if conditions or condition_tensors is not None:
                raise ValueError("pass the conditions either as conditions / condition_tensors or as the pre-computed "
                                 "cross_attention_src / prefix, not both")
        else:
            if condition_tensors is None:
                if conditions:
                    assert self.condition_provider is not None, "conditions given but the model has no condition_provider"
                    condition_tensors = self.condition_provider(self.condition_provider.tokenize(list(conditions)))
            else:
                assert not conditions, "Shouldn't pass both conditions and condition_tensors."
            if condition_tensors is not None:
                cross, prefix = self.fuser.cross_source(condition_tensors), self.fuser.prefix_source(condition_tensors)
        with torch.cuda.device(self.device):
            seq = sequence.to(self.device, torch.long).contiguous()
            # the reference's embedding lookup raises on an out-of-range token; the kernels take the range as a precondition
            if seq.numel() and not bool(((seq >= 0) & (seq <= self.card)).all()):
                raise IndexError(f"tokens must lie in [0, {self.card}] (card = the special token)")
            text_len = 0
            if self.cross_attention:
                assert cross is not None, "the model has cross attention: conditions or cross_attention_src are required"
                cross = cross.to(self.device, torch.float32).contiguous()
                assert cross.dim() == 3 and cross.shape[0] == B and cross.shape[2] == self.dim, \
                    f"cross_attention_src must be [B={B}, T, {self.dim}], got {tuple(cross.shape)}"
                text_len = cross.shape[1]
            else:
                cross = None
            prefix, P = self._check_prefix(prefix, B)
            cfg = self._config()
            nbytes = self._lib.acb_lm_forward_workspace_bytes(C.byref(cfg), B, P, S, text_len)
            if nbytes < 0:
                _lib.check(int(nbytes), 'lm_forward_workspace_bytes')
            ws = torch.empty(max(int(nbytes), 1), device=self.device, dtype=torch.uint8)
            logits = torch.empty((B, K, S, self.card), device=self.device, dtype=torch.float32)
            _lib.check(self._lib.acb_lm_forward(C.byref(cfg), C.byref(self._weights()), _lib.ptr(seq), _lib.ptr(cross),
                                                _lib.ptr(prefix), B, P, S, text_len, _lib.ptr(logits), _lib.ptr(ws),
                                                int(nbytes), _lib.stream()), 'lm_forward')
            return logits

    __call__ = forward

    @torch.no_grad()
    def compute_predictions(self, codes: torch.Tensor, conditions: tp.List[ConditioningAttributes] = [],
                            condition_tensors: tp.Optional[tp.Dict[str, tp.Any]] = None, stage: int = -1,
                            keep_only_valid_steps: bool = True, *,
                            cross_attention_src: tp.Optional[torch.Tensor] = None,
                            prefix: tp.Optional[torch.Tensor] = None) -> LMOutput:
        """LMModel.compute_predictions (lm.py:270-321): codes [B,K,T] -> LMOutput(logits [B,K,T,card], mask [B,K,T]); the
        logits of timestep t predict codes[..., t] and are NaN where the mask is 0."""
        if stage >= 0:
            raise NotImplementedError("stage >= 0 (MAGNeT's per-stage attention masks) is not built")
        B, K, T = codes.shape
        codes = codes.to(self.device).contiguous()
        pattern = self.pattern_provider.get_pattern(T)
        sequence_codes, _, _ = pattern.build_pattern_sequence(codes, self.special_token_id,
                                                              keep_only_valid_steps=keep_only_valid_steps)
        logits = self.forward(sequence_codes, conditions, condition_tensors, stage,
                              cross_attention_src=cross_attention_src, prefix=prefix)   # [B, K, S, card]
        S = logits.shape[2]
        # revert_pattern_logits' index table applied to [B, K, S, card] directly, without the [B, card, K, S] permuted copy
        idx, mask = pattern.logits_tables(S, keep_only_valid_steps)
        idx_t = torch.from_numpy(idx).to(self.device)
        flat = torch.cat([logits.reshape(B, K * S, self.card),
                          torch.full((B, 1, self.card), float('nan'), device=self.device, dtype=logits.dtype)], dim=1)
        out = flat[:, idx_t.reshape(-1)].reshape(B, K, T, self.card)
        return LMOutput(out, torch.from_numpy(mask).to(self.device)[None].expand(B, -1, -1))
