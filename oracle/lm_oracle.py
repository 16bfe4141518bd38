"""CPU oracle for the MusicGen LM decode path (LMModel.forward / _sample_next_token / generate).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Plain fp32 torch on CPU, restating the
reference algorithm with citations (paths relative to the reference source tree).  Weights come in as a
reference-layout LM ``state_dict`` (SURVEY.md section 8b).

``half_gemm=True`` emulates the GPU arithmetic of BOTH the reference GPU path (fp16 weights +
fp16 autocast, audiocraft/models/loaders.py:115-118, genmodel.py:74-78) and this repo's kernels:
weights and every GEMM input are rounded to fp16, accumulation / LayerNorm / softmax / residual stay
fp32.  ``half_gemm=False`` is the reference CPU arithmetic (everything fp32).
"""
import math
import typing as tp

import numpy as np
import torch
import torch.nn.functional as F

DEFAULT_CFG = dict(dim=1024, num_heads=16, num_layers=24, hidden_scale=4, n_q=4, card=2048,
                   delays=[0, 1, 2, 3], max_period=10000.0, positional_scale=1.0,
                   cross_attention=True, cfg_coef=3.0)


def make_cfg(**over) -> dict:
    cfg = dict(DEFAULT_CFG)
    cfg.update(over)
    return cfg


# ----------------------------------------------------------------------------- delay pattern

def delay_sequence_indexes(timesteps: int, n_q: int, delays: tp.Sequence[int]):
    """Gather table of DelayedPatternProvider.get_pattern + Pattern._build_pattern_sequence_scatter_indexes
    (audiocraft/modules/codebooks_patterns.py:339-356, 130-152): sequence step s>=1 of codebook q holds
    timestep t = s-1-delays[q] when 0 <= t < timesteps, else the special token.
    Returns (indexes [K,S] into the flattened [K*T (+1 sentinel)] codes, mask [K,S]); S = T+max_delay+1."""
    S = timesteps + max(delays) + 1
    idx = np.full((n_q, S), n_q * timesteps, dtype=np.int64)
    mask = np.zeros((n_q, S), dtype=bool)
    for q, d in enumerate(delays):
        for s in range(1, S):
            t = s - 1 - d
            if 0 <= t < timesteps:
                idx[q, s] = t + q * timesteps
                mask[q, s] = True
    return idx, mask


def build_delay_sequence(codes: torch.Tensor, delays, special: int):
    """Pattern.build_pattern_sequence. codebooks_patterns.py:154-179. codes [B,K,T] -> ([B,K,S], mask [K,S])."""
    B, K, T = codes.shape
    idx, mask = delay_sequence_indexes(T, K, delays)
    flat = torch.cat([codes.reshape(B, -1), torch.full((B, 1), special, dtype=codes.dtype)], dim=1)
    seq = flat[:, torch.from_numpy(idx).reshape(-1)].reshape(B, K, idx.shape[1])
    return seq, torch.from_numpy(mask)


def revert_delay_sequence(seq: torch.Tensor, delays, special: int, timesteps: int):
    """Pattern.revert_pattern_sequence. codebooks_patterns.py:181-248. seq [B,K,S] -> ([B,K,T], mask [K,T])."""
    B, K, S = seq.shape
    idx = np.full((K, timesteps), K * S, dtype=np.int64)
    mask = np.zeros((K, timesteps), dtype=bool)
    for q, d in enumerate(delays):
        for s in range(1, S):
            t = s - 1 - d
            if 0 <= t < timesteps:
                idx[q, t] = s + q * S
                mask[q, t] = True
    flat = torch.cat([seq.reshape(B, -1), torch.full((B, 1), special, dtype=seq.dtype)], dim=1)
    out = flat[:, torch.from_numpy(idx).reshape(-1)].reshape(B, K, timesteps)
    return out, torch.from_numpy(mask)


# ----------------------------------------------------------------------------- sampling

def multinomial(probs: torch.Tensor, generator=None) -> torch.Tensor:
    """utils.multinomial (audiocraft/utils/utils.py:88-105): torch.multinomial over the last dim, 1 sample."""
    flat = probs.reshape(-1, probs.shape[-1])
    out = torch.multinomial(flat, num_samples=1, generator=generator)
    return out.reshape(*probs.shape[:-1], 1)


def multinomial_with_noise(probs: torch.Tensor, noise: torch.Tensor) -> torch.Tensor:
    """What torch.multinomial(num_samples=1) computes: argmax(p / q), q ~ Exponential(1) drawn for every
    candidate (aten/src/ATen/native/Distributions.cpp, fast path).  With `noise` drawn as
    torch.empty_like(flat).exponential_(1, generator=g) this equals multinomial(probs, generator=g')
    for an identically-seeded g' (checked in tests/test_oracle_sampling.py)."""
    return (probs / noise.reshape(probs.shape)).argmax(dim=-1, keepdim=True)


def top_k_filter(probs: torch.Tensor, k: int) -> torch.Tensor:
    """sample_top_k up to the draw (audiocraft/utils/utils.py:108-121): keep p >= k-th largest (ties kept),
    renormalise."""
    kth = torch.topk(probs, k, dim=-1).values[..., [-1]]
    probs = probs * (probs >= kth).float()
    return probs / probs.sum(dim=-1, keepdim=True)


def top_p_sorted(probs: torch.Tensor, p: float):
    """sample_top_p up to the draw (audiocraft/utils/utils.py:125-141): returns (renormalised sorted probs,
    sort index); the draw happens in sorted space and is mapped back through the index."""
    ps, pi = torch.sort(probs, dim=-1, descending=True)
    cum = torch.cumsum(ps, dim=-1)
    ps = ps * (~(cum - ps > p)).float()
    return ps / ps.sum(dim=-1, keepdim=True), pi


def sample_from_logits(logits: torch.Tensor, use_sampling: bool, temp: float, top_k: int, top_p: float,
                       generator=None, noise: tp.Optional[torch.Tensor] = None) -> torch.Tensor:
    """Tail of LMModel._sample_next_token (audiocraft/models/lm.py:403-418). logits [B,K,card] -> [B,K,1]."""
    if not (use_sampling and temp > 0.0):
        return torch.argmax(logits, dim=-1, keepdim=True)
    probs = torch.softmax(logits / temp, dim=-1)

    def draw(p):
        return multinomial_with_noise(p, noise) if noise is not None else multinomial(p, generator)

    if top_p > 0.0:
        ps, pi = top_p_sorted(probs, top_p)
        return torch.gather(pi, -1, draw(ps))
    if top_k > 0:
        return draw(top_k_filter(probs, top_k))
    return draw(probs)


# ----------------------------------------------------------------------------- transformer

def sin_embedding(positions: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    """create_sin_embedding (audiocraft/modules/transformer.py:70-89): cat[cos, sin], divisor half_dim-1."""
    half = dim // 2
    adim = torch.arange(half, dtype=torch.float32).view(1, 1, -1)
    phase = positions.float() / (torch.tensor(max_period) ** (adim / (half - 1)))
    return torch.cat([torch.cos(phase), torch.sin(phase)], dim=-1)


def rope_rotate(x: torch.Tensor, start: int, max_period: float, scale: float) -> torch.Tensor:
    """RotaryEmbedding.rotate (audiocraft/modules/rope.py:68-69, 75-103): x [R,H,T,hd]; the head dim is hd/2 complex
    pairs (2i, 2i+1) rotated by (start + t) / max_period^(2i/hd) in fp32, blended with `scale`
    (rotation * scale + (1 - scale)), cast back to the input dtype."""
    hd, T = x.shape[-1], x.shape[2]
    adim = torch.arange(0, hd, 2, dtype=torch.float32)[: hd // 2]
    freq = 1.0 / (max_period ** (adim / hd))
    ang = torch.outer(torch.arange(start, start + T, dtype=torch.float32), freq)          # [T, hd/2]
    rot = torch.polar(torch.ones_like(ang), ang) * scale + (1.0 - scale)
    xc = torch.view_as_complex(x.float().reshape(*x.shape[:-1], -1, 2).contiguous())
    return torch.view_as_real(xc * rot.view(1, 1, T, -1)).reshape(x.shape).to(x.dtype)


class LMOracle:
    def __init__(self, state_dict: dict, cfg: dict, half_gemm: bool = False):
        self.cfg = cfg
        self.pos_emb = cfg.get('positional_embedding', 'sin')   # 'sin' | 'rope' | 'sin_rope' (transformer.py:632-637)
        self.half = half_gemm
        self.d = cfg['dim']
        self.H = cfg['num_heads']
        self.L = cfg['num_layers']
        self.K = cfg['n_q']
        self.card = cfg['card']
        sd = {}
        for k, v in state_dict.items():
            v = v.detach().cpu()
            if v.is_floating_point():
                is_matrix = v.dim() == 2
                v = v.half().float() if (half_gemm and is_matrix) else v.float()
            sd[k] = v
        self.sd = sd
        self.reset()

    # -- streaming state (StreamingModule contract, audiocraft/modules/streaming.py:20-119)
    def reset(self):
        self.kcache = [None] * self.L
        self.vcache = [None] * self.L
        self.offset = 0

    def _q(self, x):
        return x.half().float() if self.half else x

    def _lin(self, x, w):
        return F.linear(self._q(x), w)

    def _heads(self, x):  # [R,T,d] -> [R,H,T,hd]
        R, T, _ = x.shape
        return x.view(R, T, self.H, self.d // self.H).permute(0, 2, 1, 3)

    def _attend(self, q, k, v, causal_from: tp.Optional[int]):
        """softmax(q k^T / sqrt(hd)) v; what F.scaled_dot_product_attention computes at transformer.py:413.
        causal_from = number of cached steps when the multi-token first call needs the causal mask
        (transformer.py:233-264), None for single-token / cross attention."""
        hd = q.shape[-1]
        w = (self._q(q) @ self._q(k).transpose(-1, -2)) / math.sqrt(hd)
        if causal_from is not None:
            Tq, Tk = q.shape[2], k.shape[2]
            qpos = torch.arange(causal_from, causal_from + Tq).view(-1, 1)
            kpos = torch.arange(Tk).view(1, -1)
            w = w.masked_fill(kpos > qpos, float('-inf'))
        o = torch.softmax(w, dim=-1) @ self._q(v)
        R, H, T, _ = o.shape
        return self._q(o).permute(0, 2, 1, 3).reshape(R, T, H * hd)

    def _self_attn(self, li, x):
        """StreamingMultiheadAttention.forward, self-attention branch (transformer.py:362-441): packed
        in_proj laid out (p=3, h, hd) :373, KV cache append :266-298."""
        p = f'transformer.layers.{li}.self_attn.'
        proj = self._q(self._lin(x, self.sd[p + 'in_proj_weight']))
        q, k, v = [self._heads(t) for t in proj.split(self.d, dim=-1)]
        past = 0 if self.kcache[li] is None else self.kcache[li].shape[2]
        if self.pos_emb in ('rope', 'sin_rope'):
            # transformer.py:394-395 -> rope.py:106-125: q and the new k rotated at their absolute positions (the number of
            # cached keys), in fp32, cast back to the fp16 the projections are in under autocast
            q = self._q(rope_rotate(q, past, self.cfg['max_period'], self.cfg['positional_scale']))
            k = self._q(rope_rotate(k, past, self.cfg['max_period'], self.cfg['positional_scale']))
        if past:
            k = torch.cat([self.kcache[li], k], dim=2)
            v = torch.cat([self.vcache[li], v], dim=2)
        self.kcache[li], self.vcache[li] = k, v
        causal = past if x.shape[1] > 1 else None
        return self._lin(self._attend(q, k, v, causal), self.sd[p + 'out_proj.weight'])

    def _cross_attn(self, li, x, src):
        """Cross-attention branch (transformer.py:344-361): q from x with W[:d]; k, v from the condition
        with W[d:2d], W[2d:]; no padding mask is applied (the fuser drops it)."""
        p = f'transformer.layers.{li}.cross_attention.'
        w = self.sd[p + 'in_proj_weight']
        d = self.d
        q = self._heads(self._q(self._lin(x, w[:d])))
        k = self._heads(self._q(self._lin(src, w[d:2 * d])))
        v = self._heads(self._q(self._lin(src, w[2 * d:])))
        return self._lin(self._attend(q, k, v, None), self.sd[p + 'out_proj.weight'])

    def _ln(self, x, name):
        return F.layer_norm(x, (self.d,), self.sd[name + '.weight'], self.sd[name + '.bias'], 1e-5)

    def forward(self, tokens: torch.Tensor, cross_src: tp.Optional[torch.Tensor]) -> torch.Tensor:
        """LMModel.forward in streaming mode (audiocraft/models/lm.py:221-268) + StreamingTransformer.forward
        (transformer.py:693-713) + pre-norm layer (transformer.py:558-565). tokens [R,K,S] -> [R,K,S,card]."""
        R, K, S = tokens.shape
        x = sum(F.embedding(tokens[:, k], self.sd[f'emb.{k}.weight']) for k in range(K))  # [R,S,d]
        pos = (torch.arange(S).view(1, -1, 1) + self.offset)
        if self.pos_emb in ('sin', 'sin_rope'):   # transformer.py:701-705
            x = x + self.cfg['positional_scale'] * sin_embedding(pos, self.d, self.cfg['max_period'])
        for li in range(self.L):
            p = f'transformer.layers.{li}.'
            x = x + self._self_attn(li, self._ln(x, p + 'norm1'))
            if cross_src is not None:
                x = x + self._cross_attn(li, self._ln(x, p + 'norm_cross'), cross_src)
            h = self._lin(self._ln(x, p + 'norm2'), self.sd[p + 'linear1.weight'])
            x = x + self._lin(F.gelu(self._q(h)), self.sd[p + 'linear2.weight'])
        self.offset += S
        x = self._ln(x, 'out_norm')
        return torch.stack([self._lin(x, self.sd[f'linears.{k}.weight']) for k in range(K)], dim=1)

    # -- generation
    def next_token(self, seq, cross_cfg, use_sampling, temp, top_k, top_p, cfg_coef, generator, noise,
                   return_logits=False, cfg_coef_beta=None):
        """LMModel._sample_next_token, batched-CFG branch (audiocraft/models/lm.py:390-418): rows doubled
        [cond; uncond], logits = uncond + (cond - uncond) * coef, last step only."""
        B = seq.shape[0]
        if cross_cfg is not None and cfg_coef_beta is not None:
            # double CFG (lm.py:362-376): rows [cond; style-only; null]
            all_logits = self.forward(torch.cat([seq, seq, seq], dim=0), cross_cfg)
            cond, wav, uncond = all_logits.split(B, dim=0)
            logits = uncond + cfg_coef * (wav + cfg_coef_beta * (cond - wav) - uncond)
        elif cross_cfg is not None:
            all_logits = self.forward(torch.cat([seq, seq], dim=0), cross_cfg)
            cond, uncond = all_logits.split(B, dim=0)
            logits = uncond + (cond - uncond) * cfg_coef
        else:
            logits = self.forward(seq, None)
        logits = logits[:, :, -1, :]  # [B,K,card]
        tok = sample_from_logits(logits, use_sampling, temp, top_k, top_p, generator, noise)
        return (tok, logits) if return_logits else tok

    @torch.no_grad()
    def generate(self, prompt: tp.Optional[torch.Tensor], cross_cfg: tp.Optional[torch.Tensor], num_samples: int,
                 max_gen_len: int, use_sampling=True, temp=1.0, top_k=250, top_p=0.0, cfg_coef=None,
                 generator=None, noise_fn=None, record_logits: tp.Optional[list] = None,
                 teacher: tp.Optional[torch.Tensor] = None) -> torch.Tensor:
        """LMModel.generate (audiocraft/models/lm.py:420-587).  cross_cfg = [2B,Tc,d] condition rows followed by
        null rows (what condition_provider returns for conditions+null_conditions, lm.py:497-509) or None.
        noise_fn(step, shape) -> Exponential(1) noise to inject instead of a torch generator.
        teacher [B,K,S]: teacher-forced sequence (tokens taken from it instead of the sampled ones) so that
        logits of two implementations can be compared step by step."""
        cfg_coef = self.cfg['cfg_coef'] if cfg_coef is None else cfg_coef
        K, special, delays = self.K, self.card, self.cfg['delays']
        B = num_samples
        if prompt is None:
            prompt = torch.zeros((B, K, 0), dtype=torch.long)
        T0 = prompt.shape[-1]
        assert T0 < max_gen_len
        codes = torch.full((B, K, max_gen_len), -1, dtype=torch.long)
        codes[..., :T0] = prompt
        seq, mask = build_delay_sequence(codes, delays, special)
        S = seq.shape[-1]
        start = T0 + 1 + min(delays)  # Pattern.get_first_step_with_timesteps(T0), codebooks_patterns.py:119-121
        self.reset()
        prev = 0
        for offset in range(start, S):
            cur = seq[..., prev:offset]
            noise = noise_fn(offset, (B, K, self.card)) if noise_fn is not None else None
            tok, logits = self.next_token(cur, cross_cfg, use_sampling, temp, top_k, top_p, cfg_coef,
                                          generator, noise, return_logits=True)
            if record_logits is not None:
                record_logits.append(logits)
            if teacher is not None:
                tok = teacher[..., offset:offset + 1].clone()
            valid = mask[..., offset:offset + 1].expand(B, -1, -1)
            tok[~valid] = special
            here = seq[..., offset:offset + 1]
            seq[..., offset:offset + 1] = torch.where(here == -1, tok, here)
            prev = offset
        self.reset()
        assert not (seq == -1).any()
        out, out_mask = revert_delay_sequence(seq, delays, -1, max_gen_len)
        assert (out != -1).all() and out_mask.all()
        self.last_sequence = seq
        return out[..., :max_gen_len]
