"""The LM oracle with a condition prefix: the `prepend` fuser of MusicGen-melody (conditioners.py:1703-1763).

On the first streaming call the prefix vectors [rows, P, d] go in front of the token embeddings, the transformer runs
causally over [prefix ; tokens] at positions 0 .. P + S - 1 and the prefix logits are dropped (models/lm.py:265); later
calls continue at offset P + t.  ``half_gemm=True`` rounds the prefix to fp16, as the reference's autocast output_proj does
on its CUDA path; the fp32 mode uses it as given."""
import typing as tp

import torch

from oracle import lm_oracle as LO


class PrefixLMOracle(LO.LMOracle):
    def __init__(self, state_dict: dict, cfg: dict, half_gemm: bool = False, prefix: tp.Optional[torch.Tensor] = None):
        super().__init__(state_dict, cfg, half_gemm)
        self.prefix = None if prefix is None else prefix.detach().float().cpu()

    def forward(self, tokens: torch.Tensor, cross_src: tp.Optional[torch.Tensor]) -> torch.Tensor:
        """LMOracle.forward with the prefix in front on the first call.  The prefix vectors become extra rows of codebook 0's
        embedding table (zero rows in the other codebooks, so the sum over codebooks is the prefix vector exactly) and
        extra leading "tokens" that select them: the base forward then embeds, positions and runs [prefix ; tokens] as the
        fuser's concatenation does.  The prefix logits are dropped (models/lm.py:265)."""
        if self.prefix is None or self.offset != 0:
            return super().forward(tokens, cross_src)
        R, K, S = tokens.shape
        assert self.prefix.shape[0] == R, (self.prefix.shape, R)
        P = self.prefix.shape[1]
        names = [f'emb.{k}.weight' for k in range(K)]
        saved = {n: self.sd[n] for n in names}
        n0 = saved[names[0]].shape[0]
        assert all(saved[n].shape[0] == n0 for n in names)
        rows = self._q(self.prefix.reshape(R * P, self.d))
        for k, n in enumerate(names):
            self.sd[n] = torch.cat([saved[n], rows if k == 0 else torch.zeros_like(rows)])
        ptok = (n0 + torch.arange(R * P)).view(R, 1, P).expand(R, K, P)
        try:
            logits = super().forward(torch.cat([ptok, tokens], dim=2), cross_src)
        finally:
            self.sd.update(saved)
        return logits[:, :, P:]

    def next_token(self, seq, cross_cfg, use_sampling, temp, top_k, top_p, cfg_coef, generator, noise,
                   return_logits=False, cfg_coef_beta=None):
        """With a 2B-row prefix and no cross-attention source, CFG runs on the prefix rows [cond ; null]."""
        B = seq.shape[0]
        if cross_cfg is not None or self.prefix is None or self.prefix.shape[0] != 2 * B:
            return super().next_token(seq, cross_cfg, use_sampling, temp, top_k, top_p, cfg_coef, generator, noise,
                                      return_logits, cfg_coef_beta)
        cond, uncond = self.forward(torch.cat([seq, seq], dim=0), None).split(B, dim=0)
        logits = (uncond + (cond - uncond) * cfg_coef)[:, :, -1, :]
        tok = LO.sample_from_logits(logits, use_sampling, temp, top_k, top_p, generator, noise)
        return (tok, logits) if return_logits else tok

    def teacher_forced_mixed(self, seq: torch.Tensor, cross_cfg: tp.Optional[torch.Tensor], cfg_coef: float) -> torch.Tensor:
        """CFG-mixed next-token logits [S-1, B, K, card] of a known sequence [B, K, S], rows [cond ; null]."""
        B = seq.shape[0]
        self.reset()
        lg = self.forward(torch.cat([seq, seq], 0)[..., :-1], cross_cfg)
        self.reset()
        c, u = lg.split(B, dim=0)
        return (u + (c - u) * cfg_coef).permute(2, 0, 1, 3).contiguous()
