"""Generate tests/golden/encodec_tiny_gn.pt by running the REAL reference EncodecModel (found through oracle/ref_import.py:
$AUDIOCRAFT_REFERENCE or baseline/_ref) on CPU with norm='time_group_norm': GroupNorm(1, C) after every convolution
(audiocraft/modules/conv.py:33-42, 91-137).  This pins the audiocraft-format key names (`...conv.norm.*`, `...convtr.norm.*`)
and where the GroupNorm sits (before the transposed conv's trim).

    python tests/golden/make_golden_encodec_gn.py
Weights and input are regenerated from the seeds stored in the file; only outputs are stored.
"""
import os
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle.ref_models import build_ref_encodec  # noqa: E402
from tests import helpers as H  # noqa: E402
from audiocraft_b200 import synth  # noqa: E402

warnings.filterwarnings('ignore')
torch.set_grad_enabled(False)

# the tiny non-causal architecture (odd stride, dilation, two residual layers, renormalize) with GroupNorm instead of weight norm
CFG = dict(synth.ENCODEC_CONFIGS['encodec_tiny'], norm='time_group_norm')
WAV_STRIDE = 7


def main():
    batch, length, wseed, xseed = 2, 4003, 11, 12
    sd = synth.synth_encodec_state_dict(CFG, seed=wseed)
    m = build_ref_encodec(CFG, sd)
    x = H.audio_input(CFG, batch, length, xseed)
    codes, scale = m.encode(x)
    latent = m.encoder(m.preprocess(x)[0])
    wav = m.decode(codes, scale)
    out = dict(cfg=CFG, batch=batch, length=length, wseed=wseed, xseed=xseed, codes=codes, scale=scale, latent=latent,
               wav_stride=WAV_STRIDE, wav_strided=wav[..., ::WAV_STRIDE].clone(), wav_len=wav.shape[-1])
    torch.save(out, os.path.join(H.GOLDEN_DIR, 'encodec_tiny_gn.pt'))
    print('encodec_tiny_gn codes', tuple(codes.shape), 'wav', tuple(wav.shape))


if __name__ == '__main__':
    main()
