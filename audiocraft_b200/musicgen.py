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
Melody conditioning (`generate_with_chroma`, musicgen.py:155-249) runs its chroma front-end on the host once per call and
hands the LM a condition prefix; style conditioning is not built and raises.
"""
import typing as tp

import torch

from .audio_utils import convert_audio
from .conditioners import ConditioningAttributes, WavCondition
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
        ref_attributes = attributes
        while done_before_window + have < n_total:
            window_s = min(self.duration - done_before_window / fr, self.max_duration)
            attributes = self._window_attributes(ref_attributes, done_before_window / fr)
            window = self._lm_generate(prompt_tokens, attributes, int(window_s * fr), callback)
            pieces.append(window if prompt_tokens is None else window[:, :, prompt_tokens.shape[-1]:])
            prompt_tokens = window[:, :, stride:]
            have = prompt_tokens.shape[-1]
            done_before_window += stride
        return torch.cat(pieces, dim=-1)

    def _window_attributes(self, attributes, time_offset: float):
        """The conditions of the window starting `time_offset` seconds into a generation longer than max_duration."""
        return attributes


def _sampling_params(use_sampling, top_k, top_p, temperature, cfg_coef, two_step_cfg):
    return {'use_sampling': use_sampling, 'temp': temperature, 'top_k': top_k, 'top_p': top_p, 'cfg_coef': cfg_coef,
            'two_step_cfg': two_step_cfg}


class MusicGen(BaseGenModel):
    """Text-to-music (audiocraft/models/musicgen.py): 30 s window, default extension stride 18 s."""

    def __init__(self, name: str, compression_model: CompressionModel, lm: LMModel,
                 max_duration: tp.Optional[float] = None):
        super().__init__(name, compression_model, lm, max_duration)
        self.set_generation_params(duration=15)  # the reference's default duration
        if self._has_melody:   # musicgen.py:90-92: at inference the chroma is matched to the training length, unmasked
            self.lm.condition_provider.conditioners['self_wav'].match_len_on_eval = True
            self.lm.condition_provider.conditioners['self_wav']._use_masking = False

    @property
    def _has_melody(self) -> bool:
        cp = self.lm.condition_provider
        return cp is not None and 'self_wav' in cp.conditioners

    @staticmethod
    def get_pretrained(name: str = 'facebook/musicgen-medium', device=None, text_encoder=None, stem_separator=None):
        """The reference pulls checkpoints from the HF hub (musicgen.py:56-94); offline this accepts a directory holding
        the reference's exported `state_dict.bin` + `compression_state_dict.bin` (then `text_encoder` is required: a local T5
        directory in Hugging Face layout, run on the device, or a callable returning the frozen T5's hidden states and mask), or
        `synthetic/<small|medium|large|melody>` and `synthetic/stereo-<small|medium|large|melody|melody-large>` for seeded random
        weights of the released architectures (the stereo ones on the interleaved stereo codec, 8 codebooks)."""
        from .loaders import load_musicgen
        return load_musicgen(name, device=device, text_encoder=text_encoder, stem_separator=stem_separator)

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

    def generate_with_chroma(self, descriptions: tp.List[tp.Optional[str]], melody_wavs, melody_sample_rate: int,
                             progress: bool = False, return_tokens: bool = False):
        """Generate conditioned on text and melody (musicgen.py:155-189).  melody_wavs: [B,C,T], [C,T] for one
        description, or a list of [C,T] tensors / None (None: that item has a null melody)."""
        if not self._has_melody:
            raise NotImplementedError("this model has no melody ('self_wav') conditioner; use a MusicGen-melody model")
        if isinstance(melody_wavs, torch.Tensor):
            if melody_wavs.dim() == 2:
                melody_wavs = melody_wavs[None]
            if melody_wavs.dim() != 3:
                raise ValueError("Melody wavs should have a shape [B, C, T].")
            melody_wavs = list(melody_wavs)
        else:
            for melody in melody_wavs:
                if melody is not None:
                    assert melody.dim() == 2, "One melody in the list has the wrong number of dims."
        melody_wavs = [convert_audio(wav, melody_sample_rate, self.sample_rate, self.audio_channels)
                       if wav is not None else None for wav in melody_wavs]
        attributes, prompt_tokens = self._prepare_tokens_and_attributes(descriptions, None, melody_wavs)
        assert prompt_tokens is None
        tokens = self._generate_tokens(attributes, prompt_tokens, progress)
        audio = self.generate_audio(tokens)
        return (audio, tokens) if return_tokens else audio

    def _null_wav(self) -> WavCondition:
        return WavCondition(torch.zeros((1, 1, 1), device=self.device), torch.tensor([0], device=self.device),
                            sample_rate=[self.sample_rate], path=[None])

    @torch.no_grad()
    def _prepare_tokens_and_attributes(self, descriptions, prompt, melody_wavs=None):
        """musicgen.py:191-249: on a melody model every item carries a `self_wav` condition, null without a melody."""
        attributes, prompt_tokens = super()._prepare_tokens_and_attributes(descriptions, prompt)
        if melody_wavs is None:
            if self._has_melody:
                for attr in attributes:
                    attr.wav['self_wav'] = self._null_wav()
        else:
            if not self._has_melody:
                raise RuntimeError("This model doesn't support melody conditioning. Use the `melody` model.")
            assert len(melody_wavs) == len(descriptions), \
                f"number of melody wavs must match number of descriptions! " \
                f"got melody len={len(melody_wavs)}, and descriptions len={len(descriptions)}"
            for attr, melody in zip(attributes, melody_wavs):
                if melody is None:
                    attr.wav['self_wav'] = self._null_wav()
                else:
                    attr.wav['self_wav'] = WavCondition(melody[None].to(device=self.device),
                                                        torch.tensor([melody.shape[-1]], device=self.device),
                                                        sample_rate=[self.sample_rate], path=[None])
        return attributes, prompt_tokens

    def _window_attributes(self, attributes, time_offset: float):
        """musicgen.py:308-323: each window's melody is max_duration seconds of the original one from time_offset on,
        wrapped around periodically (positions % length); null melodies stay null."""
        if not self._has_melody:
            return attributes
        out = []
        for attr in attributes:
            ref = attr.wav.get('self_wav')
            attr = ConditioningAttributes(text=dict(attr.text), wav=dict(attr.wav))
            if ref is not None and int(ref.length.item()) != 0:
                wav_length = int(ref.length.item())
                initial_position = int(time_offset * self.sample_rate)
                wav_target_length = int(self.max_duration * self.sample_rate)
                positions = torch.arange(initial_position, initial_position + wav_target_length, device=self.device)
                attr.wav['self_wav'] = WavCondition(ref.wav[..., positions % wav_length],
                                                    torch.full_like(ref.length, wav_target_length),
                                                    [self.sample_rate] * ref.wav.size(0), [None], [0.])
            out.append(attr)
        return out


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
