"""Delay codebook-interleaving pattern (host logic).

Mirror of the part of ``audiocraft.modules.codebooks_patterns`` MusicGen uses: ``DelayedPatternProvider``
(codebooks_patterns.py:305-356) and the ``Pattern`` methods ``LMModel.generate`` calls (build / revert /
get_first_step_with_timesteps, :119-248).  The pattern is a closed form -- sequence step s >= 1 of codebook q
holds timestep s - 1 - delays[q] -- so the gather tables are built with vectorised numpy instead of the
reference's Python loops over a layout list.  Other providers (parallel, unroll, coarse-first, musiclm) are
out of scope: MusicGen does not use them (SURVEY.md section 2 #9).
"""
import typing as tp
from functools import lru_cache

import numpy as np
import torch


class Pattern:
    def __init__(self, timesteps: int, n_q: int, delays: tp.Sequence[int]):
        self.timesteps, self.n_q, self.delays = timesteps, n_q, list(delays)
        self.max_delay = max(self.delays)

    @property
    def num_sequence_steps(self) -> int:
        return self.timesteps + self.max_delay

    def _tables(self, timesteps: int):
        """(indexes [K,S] into flattened [K*T]+sentinel, mask [K,S]); S = pattern length incl. the special step 0."""
        S = self.timesteps + self.max_delay + 1
        s = np.arange(S)[None, :]
        d = np.asarray(self.delays)[:, None]
        t = s - 1 - d
        mask = (s >= 1) & (t >= 0) & (t < timesteps) & (t < self.timesteps)
        idx = np.where(mask, t + np.arange(self.n_q)[:, None] * timesteps, self.n_q * timesteps)
        return idx.astype(np.int64), mask

    def get_first_step_with_timesteps(self, t: int, q: tp.Optional[int] = None) -> tp.Optional[int]:
        """codebooks_patterns.py:119-121."""
        assert t <= self.timesteps
        if t >= self.timesteps:
            return None
        return t + 1 + (min(self.delays) if q is None else self.delays[q])

    def build_pattern_sequence(self, z: torch.Tensor, special_token: int, keep_only_valid_steps: bool = False):
        """codebooks_patterns.py:154-179: z [B,K,T] -> (values [B,K,S], indexes [K,S], mask [K,S])."""
        B, K, T = z.shape
        assert K == self.n_q and T <= self.timesteps
        idx, mask = self._tables(T)
        if keep_only_valid_steps:
            valid = idx.shape[1] - self.max_delay
            idx, mask = idx[:, :valid], mask[:, :valid]
        idx_t = torch.from_numpy(idx).to(z.device)
        flat = torch.cat([z.reshape(B, -1), torch.full((B, 1), special_token, dtype=z.dtype, device=z.device)], dim=1)
        values = flat[:, idx_t.reshape(-1)].reshape(B, K, idx.shape[1])
        return values, idx_t, torch.from_numpy(mask).to(z.device)

    def revert_pattern_sequence(self, s: torch.Tensor, special_token: int, keep_only_valid_steps: bool = False):
        """codebooks_patterns.py:225-248: s [B,K,S] -> (values [B,K,T], indexes [K,T], mask [K,T])."""
        B, K, S = s.shape
        assert K == self.n_q
        T = self.timesteps
        t = np.arange(T)[None, :]
        step = t + 1 + np.asarray(self.delays)[:, None]
        limit = min(S, self.timesteps + 1) if keep_only_valid_steps else S
        mask = step < limit
        idx = np.where(mask, step + np.arange(K)[:, None] * S, K * S).astype(np.int64)
        idx_t = torch.from_numpy(idx).to(s.device)
        flat = torch.cat([s.reshape(B, -1), torch.full((B, 1), special_token, dtype=s.dtype, device=s.device)], dim=1)
        values = flat[:, idx_t.reshape(-1)].reshape(B, K, T)
        return values, idx_t, torch.from_numpy(mask).to(s.device)

    def logits_tables(self, S: int, keep_only_valid_steps: bool = False):
        """_build_reverted_sequence_scatter_indexes with is_model_output=True (codebooks_patterns.py:181-223): the logits at
        sequence step s predict the token at step s + 1, so timestep t of codebook q reads step t + delays[q].  Returns
        (indexes [K,T] into the flattened [K*S] steps, K*S = the special value; mask [K,T])."""
        layout_len = self.timesteps + (0 if keep_only_valid_steps else self.max_delay) + 1
        assert S <= layout_len, f"sequence to revert is longer than the defined pattern: {S} > {layout_len}"
        t = np.arange(self.timesteps)[None, :]
        step = t + np.asarray(self.delays)[:, None]
        mask = (step < S) & (step < layout_len - 1)
        idx = np.where(mask, step + np.arange(self.n_q)[:, None] * S, self.n_q * S).astype(np.int64)
        return idx, mask

    def revert_pattern_logits(self, logits: torch.Tensor, special_token: float, keep_only_valid_steps: bool = False):
        """codebooks_patterns.py:250-269: model logits [B,card,K,S] -> (values [B,card,K,T], indexes [K,T], mask [K,T]);
        positions without a prediction hold `special_token`."""
        B, card, K, S = logits.shape
        assert K == self.n_q
        idx, mask = self.logits_tables(S, keep_only_valid_steps)
        idx_t = torch.from_numpy(idx).to(logits.device)
        flat = torch.cat([logits.reshape(B, card, -1),
                          torch.full((B, card, 1), special_token, dtype=logits.dtype, device=logits.device)], dim=-1)
        values = flat[:, :, idx_t.reshape(-1)].reshape(B, card, K, idx.shape[1])
        return values, idx_t, torch.from_numpy(mask).to(logits.device)


class DelayedPatternProvider:
    """codebooks_patterns.py:305-356 (flatten_first / empty_initial are 0 for every released MusicGen)."""

    def __init__(self, n_q: int, delays: tp.Optional[tp.List[int]] = None, flatten_first: int = 0,
                 empty_initial: int = 0):
        assert n_q > 0
        if flatten_first or empty_initial:
            raise NotImplementedError("flatten_first / empty_initial patterns are not built (unused by MusicGen)")
        self.n_q = n_q
        self.delays = list(range(n_q)) if delays is None else list(delays)
        assert len(self.delays) == n_q and sorted(self.delays) == self.delays
        self.get_pattern = lru_cache(100)(self.get_pattern)  # type: ignore

    def get_pattern(self, timesteps: int) -> Pattern:
        return Pattern(timesteps, self.n_q, self.delays)
