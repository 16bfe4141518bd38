"""Conditioning plumbing at the LM boundary (host code).

The hot path consumes ``(cond[B,T,D], mask[B,T])`` tensors, produced once per ``generate`` call: the T5 text encoder runs
in the package's kernels (``T5Conditioner``, csrc/t5.cu), the chroma front-end in host PyTorch.  This module mirrors
just the contract ``LMModel.generate`` relies on: ``ConditioningAttributes`` (conditioners.py:83-123),
``BaseConditioner`` / ``TextConditioner`` (:345-384), ``ConditioningProvider.tokenize/forward`` (:1501-1545),
``ClassifierFreeGuidanceDropout`` at p=1 as used for the null conditions (lm.py:499, conditioners.py:1427-1466) and
``ConditionFuser`` for the ``cross`` method MusicGen uses and the ``prepend`` method of MusicGen-melody (:1703-1763).
The melody front-end is here too: wav-condition collation (:1574-1610), ``WaveformConditioner`` (:518-568),
``ChromaStemConditioner`` (:571-760) and ``ChromaExtractor`` (modules/chroma.py), with the Demucs stem separation
supplied by the caller.
"""
import math
import typing as tp
from copy import deepcopy
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F
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
    mask, the output is ``output_proj(hidden) * mask`` so null rows are exact zeros.  Used with any caller-supplied encoder,
    and with seeded synthetic hidden states in tests / bench."""

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


class T5Conditioner(TextConditioner):
    """conditioners.py:422-515 on the device: transformers' T5Tokenizer on the host, then the frozen T5 encoder, output_proj
    and the mask in one acb_t5_encode call (csrc/t5.cu).  `path` is a local T5 directory in Hugging Face layout
    (audiocraft_b200.t5).  output_proj stays an nn.Linear so the LM checkpoint's `condition_provider.*` entries fill it; the
    T5 weights are kept out of the module's parameters and state dict, as the reference keeps them
    (`self.__dict__['t5']`).  Rows whose mask is all zero (None / "" entries, the whole null half of CFG) are exact zeros
    and skip the encoder.  word_dropout applies only in training, which is not built here."""

    def __init__(self, path: str, output_dim: int, finetune: bool = False, device='cuda',
                 autocast_dtype: tp.Optional[str] = 'float32', word_dropout: float = 0., normalize_text: bool = False):
        if finetune:
            raise NotImplementedError("T5Conditioner finetune=True (training T5) is not built: the encoder is frozen")
        if normalize_text:
            raise NotImplementedError("T5Conditioner normalize_text=True is not built (it needs spaCy's lemmatizer)")
        from .t5 import T5Encoder, load_tokenizer
        t5 = T5Encoder(path, device)
        super().__init__(t5.d_model, output_dim)
        self.device, self.finetune, self.word_dropout, self.normalize_text = device, finetune, word_dropout, normalize_text
        self.t5_tokenizer = load_tokenizer(path)
        self.__dict__['t5'] = t5

    def tokenize(self, x: tp.List[tp.Optional[str]]) -> tp.Dict[str, torch.Tensor]:
        entries = [xi if xi is not None else "" for xi in x]
        empty_idx = torch.LongTensor([i for i, xi in enumerate(entries) if xi == ""])
        inputs = self.t5_tokenizer(entries, return_tensors='pt', padding=True)
        inputs['attention_mask'][empty_idx, :] = 0
        return {'input_ids': inputs['input_ids'], 'attention_mask': inputs['attention_mask']}

    def forward(self, inputs: tp.Dict[str, torch.Tensor]) -> ConditionType:
        ids, mask = inputs['input_ids'], inputs['attention_mask']
        w = self.output_proj.weight
        out = torch.zeros((ids.shape[0], ids.shape[1], self.output_dim), dtype=torch.float32, device=w.device)
        live = mask.cpu().any(dim=1).nonzero().flatten()
        if len(live):
            out[live.to(w.device)] = self.t5.encode(ids[live], mask[live], w, self.output_proj.bias)[0]
        return out, mask.to(w.device)


def length_to_mask(lengths: torch.Tensor, max_len: tp.Optional[int] = None) -> torch.Tensor:
    """utils/utils.py:174-187."""
    assert len(lengths.shape) == 1, "Length shape should be 1 dimensional."
    final_length = lengths.max().item() if not max_len else max_len
    final_length = max(final_length, 1)
    return torch.arange(final_length, device=lengths.device)[None, :] < lengths[:, None]


def chroma_filter_bank(sr: int, n_fft: int, n_chroma: int = 12, tuning: float = 0.0, ctroct: float = 5.0,
                       octwidth: tp.Optional[float] = 2.0, base_c: bool = True) -> torch.Tensor:
    """The chroma filter bank [n_chroma, n_fft // 2 + 1] of ``librosa.filters.chroma`` (norm=2), restated in float64
    (librosa is not a dependency).  Every FFT bin gets a Gaussian bump around its pitch class, 2x narrower than the bin's
    width in chroma bins, each column has unit L2 norm, and the columns are weighted by a Gaussian over octaves centred on
    octave `ctroct` with standard deviation `octwidth`.  base_c: row 0 is C (otherwise A)."""
    freqs = torch.arange(1, n_fft, dtype=torch.float64) * (sr / n_fft)
    a440 = 440.0 * 2.0 ** (tuning / n_chroma)
    frqbins = n_chroma * torch.log2(freqs / (a440 / 16))                      # hz_to_octs * n_chroma
    frqbins = torch.cat([frqbins[:1] - 1.5 * n_chroma, frqbins])              # the 0 Hz bin: 1.5 octaves below bin 1
    binwidth = torch.cat([torch.clamp(frqbins[1:] - frqbins[:-1], min=1.0), torch.ones(1, dtype=torch.float64)])
    D = frqbins[None, :] - torch.arange(n_chroma, dtype=torch.float64)[:, None]
    half = float(round(n_chroma / 2))
    D = torch.remainder(D + half + 10 * n_chroma, n_chroma) - half
    wts = torch.exp(-0.5 * (2 * D / binwidth[None, :]) ** 2)
    length = torch.sqrt((wts ** 2).sum(0, keepdim=True))
    length = torch.where(length < torch.finfo(torch.float64).tiny, torch.ones_like(length), length)
    wts = wts / length
    if octwidth is not None:
        wts = wts * torch.exp(-0.5 * ((frqbins / n_chroma - ctroct) / octwidth) ** 2)[None, :]
    if base_c:
        wts = torch.roll(wts, -3 * (n_chroma // 12), dims=0)
    return wts[:, :int(1 + n_fft / 2)].to(torch.float32).contiguous()


class ChromaExtractor(nn.Module):
    """modules/chroma.py: power spectrogram (torchaudio Spectrogram: periodic Hann window, center=True with reflect padding,
    normalized=True, power 2) -> chroma filter bank -> max-normalised over the bins -> optionally one-hot of the argmax.
    wav [B,1,T] -> chroma [B, frames, n_chroma], frames = 1 + T // winhop."""

    def __init__(self, sample_rate: int, n_chroma: int = 12, radix2_exp: int = 12, nfft: tp.Optional[int] = None,
                 winlen: tp.Optional[int] = None, winhop: tp.Optional[int] = None, argmax: bool = False,
                 norm: float = torch.inf):
        super().__init__()
        self.winlen = winlen or 2 ** radix2_exp
        self.nfft = nfft or self.winlen
        self.winhop = winhop or (self.winlen // 4)
        self.sample_rate, self.n_chroma, self.norm, self.argmax = sample_rate, n_chroma, norm, argmax
        self.register_buffer('fbanks', chroma_filter_bank(sample_rate, self.nfft, n_chroma), persistent=False)
        self.register_buffer('window', torch.hann_window(self.winlen, periodic=True), persistent=False)

    def spectrogram(self, wav: torch.Tensor) -> torch.Tensor:
        shape = wav.shape
        x = wav.reshape(-1, shape[-1])
        spec = torch.stft(x, n_fft=self.nfft, hop_length=self.winhop, win_length=self.winlen, window=self.window,
                          center=True, pad_mode='reflect', normalized=False, onesided=True, return_complex=True)
        spec = spec / self.window.pow(2.0).sum().sqrt()
        spec = spec.abs().pow(2.0)
        return spec.reshape(shape[:-1] + spec.shape[-2:])

    def forward(self, wav: torch.Tensor) -> torch.Tensor:
        T = wav.shape[-1]
        if T < self.nfft:   # a nullified (1-sample) wav: pad to one FFT window
            pad = self.nfft - T
            r = 0 if pad % 2 == 0 else 1
            wav = F.pad(wav, (pad // 2, pad // 2 + r), 'constant', 0)
        spec = self.spectrogram(wav).squeeze(1)
        raw_chroma = torch.einsum('cf,...ft->...ct', self.fbanks, spec)
        norm_chroma = F.normalize(raw_chroma, p=self.norm, dim=-2, eps=1e-6).transpose(-1, -2).contiguous()
        if self.argmax:
            idx = norm_chroma.argmax(-1, keepdim=True)
            norm_chroma[:] = 0
            norm_chroma.scatter_(dim=-1, index=idx, value=1)
        return norm_chroma


class WaveformConditioner(BaseConditioner):
    """conditioners.py:518-568: a waveform -> a dense embedding -> output_proj, masked by the waveform lengths unless
    `_use_masking` is off."""

    def __init__(self, dim: int, output_dim: int, device='cpu'):
        super().__init__(dim, output_dim)
        self.device = device
        self._use_masking = True

    def tokenize(self, x: WavCondition) -> WavCondition:
        wav, length, sample_rate, path, seek_time = x
        assert length is not None
        return WavCondition(wav.to(self.device), length.to(self.device), sample_rate, path, seek_time)

    def _get_wav_embedding(self, x: WavCondition) -> torch.Tensor:
        raise NotImplementedError()

    def _downsampling_factor(self):
        raise NotImplementedError()

    def forward(self, x: WavCondition) -> ConditionType:
        wav, lengths, *_ = x
        with torch.no_grad():
            embeds = self._get_wav_embedding(x)
        if hasattr(self, 'output_proj'):
            embeds = embeds.to(self.output_proj.weight)
            embeds = self.output_proj(embeds)
        if lengths is not None and self._use_masking:
            lengths = lengths / self._downsampling_factor()
            mask = length_to_mask(lengths.to(embeds.device), max_len=embeds.shape[1]).int()
        else:
            mask = torch.ones_like(embeds[..., 0])
        embeds = embeds * mask.unsqueeze(-1)
        return embeds, mask


StemSeparator = tp.Callable[[torch.Tensor, int], torch.Tensor]


def identity_stem_separator(wav: torch.Tensor, sample_rate: int) -> torch.Tensor:
    """Stand-in for Demucs in seeded synthetic models and tests: the mono mix itself is the melody stem."""
    return wav.mean(1, keepdim=True)


class ChromaStemConditioner(WaveformConditioner):
    """conditioners.py:571-760: chroma of the melody stems (Demucs 'vocals' + 'other'), one-hot per frame with
    argmax=True, projected to the LM width.  `stem_separator(wav [B,C,T], sample_rate) -> wav [B,1,T]` at
    `sample_rate` stands in for Demucs (htdemucs weights are not bundled); the caller supplies it, as the T5 hidden
    states are supplied to PrecomputedTextConditioner.  match_len_on_eval: truncate / repeat the chroma to the
    training length `chroma_len` (frames of `duration` seconds) and do not mask."""

    def __init__(self, output_dim: int, sample_rate: int, n_chroma: int, radix2_exp: int, duration: float,
                 match_len_on_eval: bool = True, eval_wavs: tp.Optional[str] = None, n_eval_wavs: int = 0,
                 cache_path: tp.Optional[str] = None, device='cpu', stem_separator: tp.Optional[StemSeparator] = None,
                 **kwargs):
        if eval_wavs is not None:
            raise NotImplementedError("ChromaStemConditioner eval_wavs (evaluation wavs from a dataset) are not built")
        if cache_path is not None:
            raise NotImplementedError("ChromaStemConditioner cache_path (the chroma embedding cache) is not built")
        if stem_separator is None:
            raise RuntimeError("ChromaStemConditioner needs stem_separator=<callable (wav [B,C,T], sample_rate) -> melody "
                               "stems [B,1,T]> standing in for Demucs (its weights are not available offline)")
        super().__init__(dim=n_chroma, output_dim=output_dim, device=device)
        self.sample_rate = sample_rate
        self.match_len_on_eval = match_len_on_eval
        if match_len_on_eval:
            self._use_masking = False
        self.duration = duration
        self.stem_separator = stem_separator
        self.chroma = ChromaExtractor(sample_rate=sample_rate, n_chroma=n_chroma, radix2_exp=radix2_exp, **kwargs).to(device)
        self.chroma_len = self._get_chroma_len()

    def _downsampling_factor(self) -> int:
        return self.chroma.winhop

    def _get_chroma_len(self) -> int:
        dummy_wav = torch.zeros((1, int(self.sample_rate * self.duration)), device=self.fbank_device)
        return self.chroma(dummy_wav).shape[1]

    @property
    def fbank_device(self):
        return self.chroma.fbanks.device

    @torch.no_grad()
    def _compute_wav_embedding(self, wav: torch.Tensor, sample_rate: int) -> torch.Tensor:
        if wav.shape[-1] == 1:   # nullified conditions only: no stems to separate
            return self.chroma(wav)
        stems = self.stem_separator(wav, sample_rate)
        return self.chroma(stems.to(self.fbank_device, torch.float32))

    @torch.no_grad()
    def _get_wav_embedding(self, x: WavCondition) -> torch.Tensor:
        assert all(sr == x.sample_rate[0] for sr in x.sample_rate), "All sample rates in batch should be equal."
        chroma = self._compute_wav_embedding(x.wav.to(self.fbank_device), x.sample_rate[0])
        if self.match_len_on_eval:
            T = chroma.shape[1]
            if T > self.chroma_len:
                chroma = chroma[:, :self.chroma_len]
            elif T < self.chroma_len:
                chroma = chroma.repeat(1, int(math.ceil(self.chroma_len / T)), 1)[:, :self.chroma_len]
        return chroma


class ConditioningProvider(nn.Module):
    """conditioners.py:1469-1610 for text and waveform conditioners."""

    def __init__(self, conditioners: tp.Dict[str, BaseConditioner], device='cpu'):
        super().__init__()
        self.device = device
        self.conditioners = nn.ModuleDict(conditioners)

    @property
    def text_conditions(self):
        return [k for k, v in self.conditioners.items() if isinstance(v, TextConditioner)]

    @property
    def wav_conditions(self):
        return [k for k, v in self.conditioners.items() if isinstance(v, WaveformConditioner)]

    def tokenize(self, inputs: tp.List[ConditioningAttributes]) -> tp.Dict[str, tp.Any]:
        """Text conditions first, then wav conditions (the order the fuser later iterates them in)."""
        assert all(isinstance(x, ConditioningAttributes) for x in inputs), \
            "Got unexpected types input for conditioner! should be tp.List[ConditioningAttributes]"
        out = {}
        for attribute in self.text_conditions:
            out[attribute] = self.conditioners[attribute].tokenize([x.text.get(attribute) for x in inputs])
        for attribute, wav in self._collate_wavs(inputs).items():
            out[attribute] = self.conditioners[attribute].tokenize(wav)
        return out

    def _collate_wavs(self, samples: tp.List[ConditioningAttributes]) -> tp.Dict[str, WavCondition]:
        """conditioners.py:1574-1610: every sample's [1,C,T] wav -> mono, zero-padded to the longest in the batch."""
        out: tp.Dict[str, WavCondition] = {}
        for attribute in self.wav_conditions:
            wavs, lengths, srs, paths, seeks = [], [], [], [], []
            for sample in samples:
                wav, length, sample_rate, path, seek_time = sample.wav[attribute]
                assert wav.dim() == 3, f"Got wav with dim={wav.dim()}, but expected 3 [1, C, T]"
                assert wav.size(0) == 1, f"Got wav [B, C, T] with shape={wav.shape}, but expected B == 1"
                wavs.append(wav.mean(1, keepdim=True).flatten())
                lengths.append(length)
                srs.extend(sample_rate)
                paths.extend(path)
                seeks.extend(seek_time)
            stacked = torch.nn.utils.rnn.pad_sequence(wavs, batch_first=True)
            out[attribute] = WavCondition(stacked.unsqueeze(1), torch.cat([torch.as_tensor(x).reshape(-1) for x in lengths]),
                                          srs, paths, seeks)
        return out

    def forward(self, tokenized: tp.Dict[str, tp.Any]) -> tp.Dict[str, ConditionType]:
        return {k: self.conditioners[k](v) for k, v in tokenized.items()}


class ConditionFuser:
    """conditioners.py:1679-1763.  MusicGen fuses `description` by cross attention; MusicGen-melody prepends
    `[self_wav, description]` to the token embeddings (the LM prefills them into the KV cache).  `prepend` is accepted
    for those layouts, lists that contain the waveform condition `self_wav`; `sum` / `input_interpolate` are not built."""
    FUSING_METHODS = ["sum", "prepend", "cross", "ignore", "input_interpolate"]

    def __init__(self, fuse2cond: tp.Dict[str, tp.List[str]], cross_attention_pos_emb: bool = False,
                 cross_attention_pos_emb_scale: float = 1.0):
        assert all(k in self.FUSING_METHODS for k in fuse2cond.keys())
        for m in ('sum', 'prepend', 'input_interpolate'):
            if fuse2cond.get(m) and not (m == 'prepend' and 'self_wav' in fuse2cond[m]):
                raise NotImplementedError(f"fuse method '{m}' with {list(fuse2cond[m])} is not built on this path "
                                          "(only 'cross', and 'prepend' lists holding 'self_wav')")
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

    def prefix_source(self, conditions: tp.Dict[str, ConditionType]) -> tp.Optional[torch.Tensor]:
        """The `prepend` conditions, [rows, P, d]: in the order the conditions come (text before wav), each one goes in
        FRONT of what is there, so text-then-wav yields [self_wav ; description] (conditioners.py:1740-1742)."""
        assert set(conditions.keys()).issubset(set(self.cond2fuse.keys())), \
            f"given conditions contain unknown attributes for fuser, expected {self.cond2fuse.keys()}, " \
            f"got {conditions.keys()}"
        out = None
        for name, (cond, _mask) in conditions.items():
            if self.cond2fuse[name] == 'prepend':
                out = cond if out is None else torch.cat([cond, out], dim=1)
        return out
