"""`convert_audio` for the prompt path of `generate_continuation` (audiocraft/data/audio_utils.py:20-59).

Host-side preprocessing, not the hot path: a prompt is resampled once per call.  The reference delegates the
resampling to a third-party dependency that is NOT part of the reference and not a dependency here:
`julius.resample_frac` (requirements.txt:7, unpinned; algorithm restated here from julius 0.2.x `ResampleFrac`):

* reduce `old_sr/new_sr` by their gcd; cutoff `sr = rolloff * min(old, new)` with `rolloff = 0.945`, `zeros = 24`;
* for each of the `new_sr` output phases `i`, a windowed-sinc FIR over `idx = -width .. width + old_sr - 1`
  (`width = ceil(zeros * old_sr / sr)`): `t = clamp((-i / new_sr + idx / old_sr) * sr, -zeros, zeros) * pi`,
  `kernel = sinc(t) * cos(t / zeros / 2) ** 2`, normalised to unit sum (a constant signal is preserved);
* replicate-pad the input by (`width`, `width + old_sr`), one strided `conv1d` (stride `old_sr`, `new_sr` output
  channels), interleave the phases, keep `floor(new_sr * length / old_sr)` samples.

**Parity unpinned**: julius cannot be imported here, and the reference holds no golden vectors for it; the CPU tests
check the properties the construction guarantees (identity at equal rates, exact output length, constants and
band-limited sines preserved, linearity).  The channel conversion below follows `convert_audio_channels` line by line in
behaviour (audio_utils.py:20-51)."""
import math
import typing as tp

import torch
import torch.nn.functional as F


def convert_audio_channels(wav: torch.Tensor, channels: int = 2) -> torch.Tensor:
    """[..., C, T] -> [..., channels, T]: downmix to mono by averaging, replicate mono, or keep the first channels;
    anything else (fewer channels than asked for, not mono) is an error, like the reference."""
    src = wav.shape[-2]
    if src == channels:
        return wav
    if channels == 1:
        return wav.mean(dim=-2, keepdim=True)
    if src == 1:
        return wav.expand(*wav.shape[:-2], channels, wav.shape[-1])
    if src >= channels:
        return wav[..., :channels, :]
    raise ValueError('The audio file has less channels than requested but is not mono.')


def _sinc(t: torch.Tensor) -> torch.Tensor:
    return torch.where(t == 0, torch.ones_like(t), torch.sin(t) / t)


def _resample_kernels(old_sr: int, new_sr: int, zeros: int, rolloff: float) -> tp.Tuple[torch.Tensor, int]:
    sr = min(new_sr, old_sr) * rolloff
    width = math.ceil(zeros * old_sr / sr)
    idx = torch.arange(-width, width + old_sr).float()
    kernels = []
    for i in range(new_sr):
        t = ((-i / new_sr + idx / old_sr) * sr).clamp_(-zeros, zeros) * math.pi
        kernel = _sinc(t) * torch.cos(t / zeros / 2) ** 2
        kernels.append(kernel / kernel.sum())
    return torch.stack(kernels).view(new_sr, 1, -1), width


def resample_frac(x: torch.Tensor, old_sr: int, new_sr: int, zeros: int = 24, rolloff: float = 0.945) -> torch.Tensor:
    """Band-limited resampling of the last dimension by the rational factor new_sr / old_sr (see the module docstring)."""
    old_sr, new_sr = int(old_sr), int(new_sr)
    if old_sr <= 0 or new_sr <= 0:
        raise ValueError("sample rates must be positive")
    g = math.gcd(old_sr, new_sr)
    old_sr, new_sr = old_sr // g, new_sr // g
    if old_sr == new_sr:
        return x
    kernel, width = _resample_kernels(old_sr, new_sr, zeros, rolloff)
    kernel = kernel.to(device=x.device, dtype=x.dtype)
    shape, length = x.shape, x.shape[-1]
    y = F.pad(x.reshape(-1, length)[:, None], (width, width + old_sr), mode='replicate')
    y = F.conv1d(y, kernel, stride=old_sr)                       # [N, new_sr phases, frames]
    y = y.transpose(1, 2).reshape(list(shape[:-1]) + [-1])
    return y[..., :int(math.floor(new_sr * length / old_sr))]


def convert_audio(wav: torch.Tensor, from_rate: float, to_rate: float, to_channels: int) -> torch.Tensor:
    """Resample to `to_rate`, then convert the channel count (the reference's order, audio_utils.py:54-59)."""
    return convert_audio_channels(resample_frac(wav, int(from_rate), int(to_rate)), to_channels)
