"""Conditioning plumbing at the LM boundary (host code).

The hot path consumes ``(cond[B,T,D], mask[B,T])`` tensors; everything that produces them (T5, chroma, CLAP...) stays
host PyTorch / HF and runs once per ``generate`` call (SURVEY.md section 2 #12, section 8f.3).  This module mirrors
just the contract ``LMModel.generate`` relies on: ``ConditioningAttributes`` (conditioners.py:83-123),
``BaseConditioner`` / ``TextConditioner`` (:345-384), ``ConditioningProvider.tokenize/forward`` (:1501-1545),
``ClassifierFreeGuidanceDropout`` at p=1 as used for the null conditions (lm.py:499, conditioners.py:1427-1466) and
``ConditionFuser`` for the ``cross`` method MusicGen uses (:1703-1763).
"""
import typing as tp
from copy import deepcopy
from dataclasses import dataclass, field

import torch
from torch import nn

ConditionType = tp.Tuple[torch.Tensor, torch.Tensor]  # condition, mask


class WavCondition(tp.NamedTuple):
    wav: torch.Tensor
    length: torch.Tensor
    sample_rate: tp.List[int]
    path: tp.List[tp.Optional[str]] = []
    seek_time: tp.List[tp.Optional[float]] = []


@dataclass
class ConditioningAttributes:
    text: tp.Dict[str, tp.Optional[str]] = field(default_factory=dict)
    wav: tp.Dict[str, WavCondition] = field(default_factory=dict)

    def __getitem__(self, item):
        return getattr(self, item)

    @property
    def text_attributes(self):
        return self.text.keys()

    @property
    def wav_attributes(self):
        return self.wav.keys()


def nullify_all(samples: tp.List[ConditioningAttributes]) -> tp.List[ConditioningAttributes]:
    """ClassifierFreeGuidanceDropout(p=1.0)(conditions): every text attribute -> None, every wav -> null wav."""
    out = deepcopy(samples)
    for s in out:
        for k in list(s.text.keys()):
            s.text[k] = None
        for k, w in list(s.wav.items()):
            s.wav[k] = WavCondition(torch.zeros_like(w.wav[..., :1]), torch.zeros_like(w.length), w.sample_rate,
                                    [None] * len(w.path), [None] * len(w.seek_time))
    return out


class BaseConditioner(nn.Module):
    """conditioners.py:345-380."""

    def __init__(self, dim: int, output_dim: int):
        super().__init__()
        self.dim, self.output_dim = dim, output_dim
        if output_dim > -1:
            self.output_proj = nn.Linear(dim, output_dim)

    def tokenize(self, *args, **kwargs) -> tp.Any:
        raise NotImplementedError()

    def forward(self, inputs: tp.Any) -> ConditionType:
        raise NotImplementedError()


class TextConditioner(BaseConditioner):
    ...


class PrecomputedTextConditioner(TextConditioner):
    """Text conditioner whose encoder output is supplied by the caller: ``encoder(list[str]) -> (hidden [B,T,dim],
    mask [B,T])``.  It reproduces T5Conditioner's contract (conditioners.py:490-515): None / "" entries get a zero
    mask, the output is ``output_proj(hidden) * mask`` so null rows are exact zeros.  Used with a T5 encoder when its
    weights are present, and with seeded synthetic hidden states in tests / bench (no network in this image)."""

    def __init__(self, dim: int, output_dim: int, encoder: tp.Callable[[tp.List[str]], ConditionType]):
        super().__init__(dim, output_dim)
        self.encoder = encoder

    def tokenize(self, x: tp.List[tp.Optional[str]]):
        entries = [xi if xi is not None else "" for xi in x]
        hidden, mask = self.encoder(entries)
        mask = mask.clone()
        empty = [i for i, e in enumerate(entries) if e == ""]
        if empty:
            mask[empty, :] = 0
        return {'hidden': hidden, 'attention_mask': mask}

    def forward(self, inputs) -> ConditionType:
        w = self.output_proj.weight
        mask = inputs['attention_mask'].to(w.device)
        embeds = self.output_proj(inputs['hidden'].to(w))
        return embeds * mask.unsqueeze(-1).to(embeds.dtype), mask


class ConditioningProvider(nn.Module):
    """conditioners.py:1469-1545 for text conditioners."""

    def __init__(self, conditioners: tp.Dict[str, BaseConditioner], device='cpu'):
        super().__init__()
        self.device = device
        self.conditioners = nn.ModuleDict(conditioners)

    @property
    def text_conditions(self):
        return [k for k, v in self.conditioners.items() if isinstance(v, TextConditioner)]

    def tokenize(self, inputs: tp.List[ConditioningAttributes]) -> tp.Dict[str, tp.Any]:
        assert all(isinstance(x, ConditioningAttributes) for x in inputs), \
            "Got unexpected types input for conditioner! should be tp.List[ConditioningAttributes]"
        out = {}
        for attribute in self.text_conditions:
            out[attribute] = self.conditioners[attribute].tokenize([x.text.get(attribute) for x in inputs])
        return out

    def forward(self, tokenized: tp.Dict[str, tp.Any]) -> tp.Dict[str, ConditionType]:
        return {k: self.conditioners[k](v) for k, v in tokenized.items()}


class ConditionFuser:
    """conditioners.py:1679-1763.  MusicGen fuses `description` by cross attention; `sum` / `prepend` /
    `input_interpolate` need a prefill path and are not built (section 8f)."""
    FUSING_METHODS = ["sum", "prepend", "cross", "ignore", "input_interpolate"]

    def __init__(self, fuse2cond: tp.Dict[str, tp.List[str]], cross_attention_pos_emb: bool = False,
                 cross_attention_pos_emb_scale: float = 1.0):
        assert all(k in self.FUSING_METHODS for k in fuse2cond.keys())
        for m in ('sum', 'prepend', 'input_interpolate'):
            if fuse2cond.get(m):
                raise NotImplementedError(f"fuse method '{m}' is not built on this path (only 'cross')")
        if cross_attention_pos_emb:
            raise NotImplementedError("cross_attention_pos_emb is not built (false for MusicGen)")
        self.fuse2cond = fuse2cond
        self.cond2fuse = {c: m for m, cs in fuse2cond.items() for c in cs}

    def cross_source(self, conditions: tp.Dict[str, ConditionType]) -> tp.Optional[torch.Tensor]:
        assert set(conditions.keys()).issubset(set(self.cond2fuse.keys())), \
            f"given conditions contain unknown attributes for fuser, expected {self.cond2fuse.keys()}, " \
            f"got {conditions.keys()}"
        out = None
        for name, (cond, _mask) in conditions.items():
            if self.cond2fuse[name] == 'cross':
                out = cond if out is None else torch.cat([out, cond], dim=1)
        return out
