"""Generation API on H100: `MusicGen` / `AudioGen` with the reference's public surface.

Behavioural contract (what callers of `audiocraft.models.MusicGen` / `AudioGen` / `BaseGenModel` rely on,
audiocraft/models/genmodel.py:28-267, musicgen.py:41-338, audiogen.py:23-93):

* `generate(descriptions)`, `generate_unconditional(n)`, `generate_continuation(prompt, sr, descriptions)` return a
  waveform `[B, C, T]` (and the token tensor `[B, K, T_frames]` first-class when `return_tokens=True`);
* `set_generation_params(...)` stores the sampling options handed to `LMModel.generate` and the target `duration`;
  `duration * frame_rate` tokens are produced (truncating), and a duration beyond `max_duration` is produced window by
  window: every window re-generates with the last `max_duration - extend_stride` seconds of tokens as its prompt;
* `progress=True` reports `(tokens_done, tokens_total)` to the custom callback or prints it;
* `generate_audio(tokens)` is the codec decode, without trimming the decoder's extra padding.

Everything here is host glue; the two hot loops live behind `LMModel.generate` and `CompressionModel.decode`.
Melody / style conditioning are conditioner front-ends outside the hot path (SURVEY.md section 8f.3) and raise.
"""
import typing as tp

import torch

from .audio_utils import convert_audio
from .conditioners import ConditioningAttributes
from .encodec import CompressionModel
from .lm import LMModel

Waveform = torch.Tensor
Tokens = torch.Tensor


class BaseGenModel:
    def __init__(self, name: str, compression_model: CompressionModel, lm: LMModel,
                 max_duration: tp.Optional[float] = None):
        if max_duration is None:
            raise ValueError("You must provide max_duration when building directly your GenModel")
        self.name, self.compression_model, self.lm = name, compression_model.eval(), lm.eval()
        # a code >= bins (or the LM's special token) must never reach the codec: the reference would raise an index error
        assert lm.card == compression_model.cardinality, \
            f"LM cardinality {lm.card} != codec cardinality {compression_model.cardinality}"
        assert lm.n_q == compression_model.num_codebooks, \
            f"LM codebooks {lm.n_q} != codec codebooks {compression_model.num_codebooks}"
        self.cfg = None
        self.device = lm.device
        self.max_duration = float(max_duration)
        self.duration = self.max_duration
        self.extend_stride: tp.Optional[float] = None
        self.generation_params: tp.Dict[str, tp.Any] = {}
        self._progress_callback: tp.Optional[tp.Callable[[int, int], None]] = None

    # -- codec facts the callers read
    frame_rate = property(lambda self: self.compression_model.frame_rate)
    sample_rate = property(lambda self: self.compression_model.sample_rate)
    audio_channels = property(lambda self: self.compression_model.channels)

    def set_custom_progress_callback(self, progress_callback=None):
        self._progress_callback = progress_callback

    # -- public generation entry points: all funnel into _run
    def generate_unconditional(self, num_samples: int, progress: bool = False, return_tokens: bool = False):
        return self._run([None] * num_samples, None, progress, return_tokens)

    def generate(self, descriptions: tp.List[str], progress: bool = False, return_tokens: bool = False):
        return self._run(descriptions, None, progress, return_tokens)

    def generate_continuation(self, prompt: Waveform, prompt_sample_rate: int,
                              descriptions: tp.Optional[tp.List[tp.Optional[str]]] = None, progress: bool = False,
                              return_tokens: bool = False):
        if prompt.dim() == 2:
            prompt = prompt[None]
        if prompt.dim() != 3:
            raise ValueError("prompt should have 3 dimensions: [B, C, T] (C = 1).")
        # resample / remix like the reference (genmodel.py:183 -> data/audio_utils.py:54-59); host-side, once per call
        prompt = convert_audio(prompt, prompt_sample_rate, self.sample_rate, self.audio_channels)
        if descriptions is None:
            descriptions = [None] * len(prompt)
        return self._run(descriptions, prompt, progress, return_tokens)

    def generate_audio(self, gen_tokens: Tokens) -> Waveform:
        assert gen_tokens.dim() == 3
        with torch.no_grad():
            return self.compression_model.decode(gen_tokens, None)

    # -- internals
    def _run(self, descriptions, prompt_wav, progress, return_tokens):
        attributes, prompt_tokens = self._prepare_tokens_and_attributes(descriptions, prompt_wav)
        tokens = self._generate_tokens(attributes, prompt_tokens, progress)
        audio = self.generate_audio(tokens)
        return (audio, tokens) if return_tokens else audio

    @torch.no_grad()
    def _prepare_tokens_and_attributes(self, descriptions: tp.Sequence[tp.Optional[str]],
                                       prompt: tp.Optional[Waveform]):
        attributes = [ConditioningAttributes(text={'description': d}) for d in descriptions]
        if prompt is None:
            return attributes, None
        assert len(descriptions) == len(prompt), "Prompt and nb. descriptions doesn't match"
        prompt_tokens, scale = self.compression_model.encode(prompt.to(self.device))
        assert scale is None
        return attributes, prompt_tokens

    def _lm_generate(self, prompt_tokens, attributes, n_tokens, callback):
        return self.lm.generate(prompt_tokens, attributes, callback=callback, max_gen_len=n_tokens, **self.generation_params)

    def _generate_tokens(self, attributes, prompt_tokens: tp.Optional[Tokens], progress: bool = False) -> Tokens:
        fr = self.frame_rate
        n_total = int(self.duration * fr)
        done_before_window = 0

        def report(done_in_window: int, total_in_window: int):
            done = done_before_window + done_in_window
            if self._progress_callback is not None:
                self._progress_callback(done, total_in_window)
            else:
                print(f'{done: 6d} / {total_in_window: 6d}', end='\r')

        callback = report if progress else None
        if prompt_tokens is not None:
            assert int(min(self.duration, self.max_duration) * fr) >= prompt_tokens.shape[-1], \
                "Prompt is longer than audio to generate"
        if self.duration <= self.max_duration:
            return self._lm_generate(prompt_tokens, attributes, n_total, callback)

        # longer than the model's window: slide by `extend_stride`, each window prompted with the tail of the previous
        assert self.extend_stride is not None, "Stride should be defined to generate beyond max_duration"
        assert self.extend_stride < self.max_duration, "Cannot stride by more than max generation duration."
        stride = int(fr * self.extend_stride)
        pieces: tp.List[Tokens] = [] if prompt_tokens is None else [prompt_tokens]
        have = 0 if prompt_tokens is None else prompt_tokens.shape[-1]
        while done_before_window + have < n_total:
            window_s = min(self.duration - done_before_window / fr, self.max_duration)
            window = self._lm_generate(prompt_tokens, attributes, int(window_s * fr), callback)
            pieces.append(window if prompt_tokens is None else window[:, :, prompt_tokens.shape[-1]:])
            prompt_tokens = window[:, :, stride:]
            have = prompt_tokens.shape[-1]
            done_before_window += stride
        return torch.cat(pieces, dim=-1)


def _sampling_params(use_sampling, top_k, top_p, temperature, cfg_coef, two_step_cfg):
    return {'use_sampling': use_sampling, 'temp': temperature, 'top_k': top_k, 'top_p': top_p, 'cfg_coef': cfg_coef,
            'two_step_cfg': two_step_cfg}


class MusicGen(BaseGenModel):
    """Text-to-music (audiocraft/models/musicgen.py): 30 s window, default extension stride 18 s."""

    def __init__(self, name: str, compression_model: CompressionModel, lm: LMModel,
                 max_duration: tp.Optional[float] = None):
        super().__init__(name, compression_model, lm, max_duration)
        self.set_generation_params(duration=15)  # the reference's default duration

    @staticmethod
    def get_pretrained(name: str = 'facebook/musicgen-medium', device=None, text_encoder=None):
        """The reference pulls checkpoints from the HF hub (musicgen.py:56-94); offline this accepts a directory holding
        the reference's exported `state_dict.bin` + `compression_state_dict.bin` (then `text_encoder`, a callable returning
        the frozen T5's hidden states and mask, is required: T5 is outside the hot path and not available offline), or
        `synthetic/<small|medium|large>` for seeded random weights of the released architectures."""
        from .loaders import load_musicgen
        return load_musicgen(name, device=device, text_encoder=text_encoder)

    def set_generation_params(self, use_sampling: bool = True, top_k: int = 250, top_p: float = 0.0,
                              temperature: float = 1.0, duration: float = 30.0, cfg_coef: float = 3.0,
                              cfg_coef_beta: tp.Optional[float] = None, two_step_cfg: bool = False,
                              extend_stride: float = 18):
        assert extend_stride < self.max_duration, "Cannot stride by more than max generation duration."
        self.extend_stride, self.duration = extend_stride, duration
        self.generation_params = _sampling_params(use_sampling, top_k, top_p, temperature, cfg_coef, two_step_cfg)
        self.generation_params['cfg_coef_beta'] = cfg_coef_beta

    def set_style_conditioner_params(self, *args, **kwargs):
        raise NotImplementedError("MusicGen-Style conditioning is not built on this path (SURVEY.md 8f.3)")

    def generate_with_chroma(self, *args, **kwargs):
        raise NotImplementedError("melody (chroma) conditioning is not built on this path (SURVEY.md 8f.3)")


class AudioGen(BaseGenModel):
    """Text-to-sound (audiocraft/models/audiogen.py:23-93): the same LM decode + EnCodec decode path at 16 kHz (codec
    `encodec_large_nq4_s320`, 4 codebooks, delays [0,1,2,3]); 10 s window, default stride 2 s, default duration 5 s."""

    def __init__(self, name: str, compression_model: CompressionModel, lm: LMModel,
                 max_duration: tp.Optional[float] = None):
        super().__init__(name, compression_model, lm, max_duration)
        self.set_generation_params(duration=5)

    @staticmethod
    def get_pretrained(name: str = 'facebook/audiogen-medium', device=None, text_encoder=None):
        from .loaders import load_audiogen
        return load_audiogen(name, device=device, text_encoder=text_encoder)

    def set_generation_params(self, use_sampling: bool = True, top_k: int = 250, top_p: float = 0.0,
                              temperature: float = 1.0, duration: float = 10.0, cfg_coef: float = 3.0,
                              two_step_cfg: bool = False, extend_stride: float = 2):
        assert extend_stride < self.max_duration, "Cannot stride by more than max generation duration."
        self.extend_stride, self.duration = extend_stride, duration
        self.generation_params = _sampling_params(use_sampling, top_k, top_p, temperature, cfg_coef, two_step_cfg)
