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
from dataclasses import dataclass

import torch

from .audio_utils import convert_audio
from .conditioners import ConditioningAttributes, WavCondition
from .encodec import CompressionModel
from .lm import LMModel

Waveform = torch.Tensor
Tokens = torch.Tensor


@dataclass(frozen=True)
class Window:
    """One LM window of a generation: it generates `length` frames, its first `prompt_len` given (already part of the output),
    starts `start` frames (`time_offset` seconds) into the generation, and its frames from `stride` on are the next window's
    prompt."""
    length: int
    prompt_len: int
    start: int
    time_offset: float
    stride: int


def window_plan(duration: float, max_duration: float, extend_stride: tp.Optional[float], frame_rate: float,
                prompt_len: int = 0) -> tp.List[Window]:
    """The windows of a generation of `duration` seconds from a prompt of `prompt_len` frames, as `_token_windows` runs
    them: one window of int(duration * frame_rate) frames up to max_duration; past it, windows of at most max_duration
    seconds, each starting int(frame_rate * extend_stride) frames after the previous one and prompted with the previous
    window's frames from that stride on, until int(duration * frame_rate) frames are produced."""
    n_total = int(duration * frame_rate)
    if duration <= max_duration:
        return [Window(n_total, prompt_len, 0, 0.0, 0)]
    assert extend_stride is not None, "Stride should be defined to generate beyond max_duration"
    assert extend_stride < max_duration, "Cannot stride by more than max generation duration."
    stride = int(frame_rate * extend_stride)
    plan, done, have = [], 0, prompt_len
    while done + have < n_total:
        length = int(min(duration - done / frame_rate, max_duration) * frame_rate)
        plan.append(Window(length, have, done, done / frame_rate, stride))
        have = max(0, length - stride)
        done += stride
    return plan


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
        def window(prompt, attrs, n, callback):
            yield self._lm_generate(prompt, attrs, n, callback)
        return torch.cat(list(self._token_windows(attributes, prompt_tokens, progress, window)), dim=-1)

    def _token_windows(self, attributes, prompt_tokens: tp.Optional[Tokens], progress: bool, window) -> tp.Iterator[Tokens]:
        """The window loop of a generation: yields token pieces whose concatenation is the generation's tokens.
        `window(prompt, attributes, n_tokens, callback)` runs the LM on one window and yields that window's tokens (its prompt
        included) in one or more pieces; past max_duration each window's new frames are yielded as they arrive."""
        fr = self.frame_rate
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
        plan = window_plan(self.duration, self.max_duration, self.extend_stride, fr,
                           0 if prompt_tokens is None else prompt_tokens.shape[-1])
        if self.duration <= self.max_duration:
            yield from window(prompt_tokens, attributes, plan[0].length, callback)
            return

        # longer than the model's window: slide by `extend_stride`, each window prompted with the tail of the previous
        if prompt_tokens is not None:
            yield prompt_tokens
        ref_attributes = attributes
        for w in plan:
            done_before_window = w.start
            attributes = self._window_attributes(ref_attributes, w.time_offset)
            skip = w.prompt_len   # the window's prompt was yielded already
            got: tp.List[Tokens] = []
            seen = 0
            for piece in window(prompt_tokens, attributes, w.length, callback):
                got.append(piece)
                new = piece[:, :, max(0, skip - seen):]
                seen += piece.shape[-1]
                if new.shape[-1]:
                    yield new
            prompt_tokens = torch.cat(got, dim=-1)[:, :, w.stride:]

    def _window_attributes(self, attributes, time_offset: float):
        """The conditions of the window starting `time_offset` seconds into a generation longer than max_duration."""
        return attributes

    # -- streaming
    def generate_stream(self, descriptions: tp.Optional[tp.List[tp.Optional[str]]] = None, *,
                        num_samples: tp.Optional[int] = None, prompt: tp.Optional[Waveform] = None,
                        prompt_sample_rate: tp.Optional[int] = None, melody_wavs=None,
                        melody_sample_rate: tp.Optional[int] = None, chunk_duration: float = 1.0, progress: bool = False,
                        return_tokens: bool = False) -> tp.Iterator[tp.Any]:
        """Generate and decode at the same time: yields waveform pieces [B, C, m] (or (wav, tokens) pairs with return_tokens)
        as the LM produces frames.  Their concatenation is what `generate` (descriptions), `generate_unconditional`
        (num_samples), `generate_continuation` (prompt) or `generate_with_chroma` (melody_wavs) returns for the same inputs and
        seed; a continuation's first pieces are the prompt's audio, as that output contains it.  The LM runs
        `chunk_duration` seconds of decode steps at a time and each block's finished frames go to the codec's stream decoder;
        the last piece holds the decoder's tail."""
        if not chunk_duration > 0:
            raise ValueError(f"chunk_duration must be > 0, got {chunk_duration}")
        if not hasattr(self.compression_model, 'stream_decoder'):
            raise NotImplementedError(f"{type(self.compression_model).__name__} has no stream decoder")
        if prompt is not None and melody_wavs is not None:
            raise ValueError("a prompt and melody_wavs together: generate_with_chroma takes no prompt")
        if descriptions is None:
            descriptions = [None] * (num_samples if num_samples is not None else
                                     (len(prompt) if prompt is not None and prompt.dim() == 3 else 1))
        # the codec refuses before any device work (GroupNorm / transformers checkpoints)
        decoder = self.compression_model.stream_decoder(len(descriptions))
        if prompt is not None:
            if prompt.dim() == 2:
                prompt = prompt[None]
            if prompt.dim() != 3:
                raise ValueError("prompt should have 3 dimensions: [B, C, T] (C = 1).")
            if prompt_sample_rate is None:
                raise ValueError("prompt_sample_rate is required with a prompt")
            prompt = convert_audio(prompt, prompt_sample_rate, self.sample_rate, self.audio_channels)
        if melody_wavs is not None:
            attributes, prompt_tokens = self._prepare_melody(descriptions, melody_wavs, melody_sample_rate)
        else:
            attributes, prompt_tokens = self._prepare_tokens_and_attributes(descriptions, prompt)
        block = max(1, int(round(chunk_duration * self.frame_rate)))

        def window(prompt_, attrs, n, callback):
            return self.lm.generate_blocks(prompt_, attrs, callback=callback, max_gen_len=n, block=block,
                                           **self.generation_params)

        with torch.no_grad():
            for tokens in self._token_windows(attributes, prompt_tokens, progress, window):
                for t0 in range(0, tokens.shape[-1], block):   # a prompt is handed to the codec in blocks too
                    piece = tokens[:, :, t0:t0 + block]
                    wav = decoder.push(piece)
                    if wav.shape[-1] or return_tokens:
                        yield (wav, piece) if return_tokens else wav
            wav = decoder.flush()
            empty = torch.empty((len(descriptions), self.lm.n_q, 0), dtype=torch.long, device=self.device)
            yield (wav, empty) if return_tokens else wav

    def _prepare_melody(self, descriptions, melody_wavs, melody_sample_rate):
        raise NotImplementedError("this model has no melody ('self_wav') conditioner; use a MusicGen-melody model")

    # -- continuous batching
    def continuous(self, slots: int = 32, poll_steps: tp.Optional[int] = None, max_text: int = 64,
                   return_tokens: bool = False, chunk_duration: tp.Optional[float] = None,
                   kv_cache_gb: tp.Optional[float] = None, prefill_prompts: bool = False, kv_cache_dtype: str = 'fp16'):
        """A `batching.ContinuousGenerator` over this model: up to `slots` requests decode side by side, each admitted when a
        slot frees and retired when its last frame is sampled.  `submit(description, duration, prompt, prompt_sample_rate,
        use_sampling=, top_k=, top_p=, temperature=, cfg_coef=)` returns a request id (options left out take the current
        generation parameters) and `cancel(request_id)` stops a request.  `poll()` / `run()` return `(request_id, wav[, tokens])`
        as requests finish, each equal to that request generated alone; with `chunk_duration` (seconds of decode steps per
        round) they return `(request_id, piece[, tokens], final)` audio pieces while the requests decode.  `max_text` bounds a
        description's text positions.  On a melody model `submit(..., melody=, melody_sample_rate=)` conditions a request on
        its melody as `generate_with_chroma` does (no melody: a null one); each request's chroma and description prefix is
        prefilled into its slot when it is admitted.

        `kv_cache_gb` (None: every slot reserves the KV cache of the longest request) is a budget in GB (1e9 bytes) for the
        self-attention KV cache: a pool of floor(kv_cache_gb * 1e9 / page_bytes) pages of 64 positions, page_bytes = 64 x
        4 x num_layers x dim bytes, from which each request takes only the pages its own length needs; a request waits until
        a slot and its pages are free.  The budget covers that pool only.  The session also allocates the cross-attention
        K/V for 2 x slots x max_text positions, a staging cache of 2 x (chroma + description) positions for admitting a
        melody prefix, and the split-K partial sums (`part`, 16 x the padded rows x max(3 dim, ffn, n_q x card) fp32).  A
        request's result is the same with or without a budget.

        `prefill_prompts` (default False: a continuation prompt is consumed one decode step per frame, and results equal
        `generate` with ACB_LM_PREFILL=0) prefills each request's prompt into its slot at admission, as `generate` prefills
        it, so results equal `generate`'s default path; it also serves durations beyond max_duration window by window, as
        `generate` does (not with chunk_duration).  The passes stall every slot while they run: it lowers a prompted
        request's latency and can cost throughput in a busy session (see `batching.ContinuousGenerator`).

        `kv_cache_dtype='fp8'` (with kv_cache_gb only) stores the paged self-attention cache in FP8: each K or V vector of
        64 values (one position of one head of one layer in one row) is 64 e4m3 codes plus one fp32 scale, page_bytes =
        64 x num_layers x (2 dim + 8 num_heads), about 1.88x the pages of an fp16 pool in the same budget.  A vector x, the
        fp32 value the fp16 cache rounds to fp16 (after rotary positions for K), is stored as amax = max |x_j|, code_j =
        e4m3(x_j * (448 / amax)) rounded to nearest even and saturated at +-448, scale = amax / 448 (both divisions
        correctly rounded; amax = 0 stores zeros), and every read of the cache sees code x scale.  Decode steps and prompt
        prefill quantize their own K/V; a melody prefix is prefilled into an fp16 staging cache, then quantized into the
        request's pages.  Cross-attention K/V, queries, activations and weights stay as they are.  Results then differ from
        `generate` and from the fp16 session; since quantization is local to one row and position, each request's result
        still equals that request alone in an fp8 session.  Refused before any device work (ValueError): any other
        kv_cache_dtype, and 'fp8' without kv_cache_gb."""
        from .batching import ContinuousGenerator
        return ContinuousGenerator(self, slots, poll_steps, max_text, return_tokens, chunk_duration, kv_cache_gb,
                                   prefill_prompts, kv_cache_dtype)


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
    def get_pretrained(name: str = 'facebook/musicgen-medium', device=None, text_encoder=None, stem_separator=None,
                       weight_dtype: str = 'fp16'):
        """The reference pulls checkpoints from the HF hub (musicgen.py:56-94); offline this accepts a directory holding
        the reference's exported `state_dict.bin` + `compression_state_dict.bin` (then `text_encoder` is required: a local T5
        directory in Hugging Face layout, run on the device, or a callable returning the frozen T5's hidden states and mask), or
        `synthetic/<small|medium|large|melody>` and `synthetic/stereo-<small|medium|large|melody|melody-large>` for seeded random
        weights of the released architectures (the stereo ones on the interleaved stereo codec, 8 codebooks).
        `weight_dtype='fp8'` quantizes the LM's per-layer matrices to e4m3 with fp32 row scales at load (LMModel)."""
        from .loaders import load_musicgen
        return load_musicgen(name, device=device, text_encoder=text_encoder, stem_separator=stem_separator,
                             weight_dtype=weight_dtype)

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
        attributes, prompt_tokens = self._prepare_melody(descriptions, melody_wavs, melody_sample_rate)
        assert prompt_tokens is None
        tokens = self._generate_tokens(attributes, prompt_tokens, progress)
        audio = self.generate_audio(tokens)
        return (audio, tokens) if return_tokens else audio

    def _prepare_melody(self, descriptions, melody_wavs, melody_sample_rate):
        """generate_with_chroma's inputs -> (attributes, prompt tokens = None) (musicgen.py:155-189)."""
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
        return self._prepare_tokens_and_attributes(descriptions, None, melody_wavs)

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
    def get_pretrained(name: str = 'facebook/audiogen-medium', device=None, text_encoder=None, weight_dtype: str = 'fp16'):
        from .loaders import load_audiogen
        return load_audiogen(name, device=device, text_encoder=text_encoder, weight_dtype=weight_dtype)

    def set_generation_params(self, use_sampling: bool = True, top_k: int = 250, top_p: float = 0.0,
                              temperature: float = 1.0, duration: float = 10.0, cfg_coef: float = 3.0,
                              two_step_cfg: bool = False, extend_stride: float = 2):
        assert extend_stride < self.max_duration, "Cannot stride by more than max generation duration."
        self.extend_stride, self.duration = extend_stride, duration
        self.generation_params = _sampling_params(use_sampling, top_k, top_p, temperature, cfg_coef, two_step_cfg)
