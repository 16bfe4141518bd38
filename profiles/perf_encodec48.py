"""EnCodec 48 kHz (stereo, GroupNorm, 1 s chunks with overlap-add): encode + decode of B x 10 s through
`HFEncodecCompressionModel.model.encode / .decode` on the kernels, against transformers' fp32 eager EncodecModel on the same
GPU with the same seeded weights.  CUDA events after a warm-up; a separate torch.profiler pass gives the GroupNorm kernels'
share of device time and their achieved HBM bandwidth (bytes computed from the shapes each call sees).

    python profiles/perf_encodec48.py [--batches 1 8 32] [--seconds 10] [--iters 3]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200.encodec import HFEncodecCompressionModel  # noqa: E402
from tests.encodec_gn_oracle import hf_48k_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--batches', type=int, nargs='+', default=[1, 8, 32])
ap.add_argument('--seconds', type=float, default=10.0)
ap.add_argument('--iters', type=int, default=3)
ap.add_argument('--bandwidth', type=float, default=24.0)
ap.add_argument('--no-transformers', action='store_true')
a = ap.parse_args()
assert torch.cuda.is_available(), 'this measurement needs the GPU'

card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                      capture_output=True, text=True).stdout.strip().splitlines()
print(f'GPU: {torch.cuda.get_device_name()} | nvidia-smi name, power limit, max SM clock: {card[0] if card else "n/a"}')

# transformers in fp32: no TF32 in its convolutions or matmuls
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
hf = hf_48k_model(seed=0)
m = HFEncodecCompressionModel(hf.state_dict(), hf.config)
hf = hf.cuda()
sr = 48000


def run_ours(x):
    codes, scales, pad = m.model.encode(x, None, a.bandwidth)
    return m.model.decode(codes, scales, None, pad)[0]


@torch.no_grad()
def run_hf(x):
    codes, scales, pad = hf.encode(x, None, a.bandwidth, return_dict=False)
    return hf.decode(codes, scales, None, False, pad)[0]


def timed(fn, x):
    fn(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        fn(x)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.iters / 1e3


gn_bytes = []
_stats, _apply = m._gn_stats, m._gn_apply


def stats_logged(y):
    gn_bytes.append(y.numel() * 4)                                    # one read of the layer output
    return _stats(y)


def apply_logged(y, L, st, left=0, t_out=None, add=None):
    out = _apply(y, L, st, left, t_out, add)
    gn_bytes.append(out.numel() * 4 * (3 if add is not None else 2))  # window read (+ second input) + write
    return out


print(f'{"B":>3s} {"audio s":>8s} {"ours s":>8s} {"hf s":>8s} {"speedup":>8s} {"ours audio-s/s":>15s} {"ours MS/s":>10s} '
      f'{"GN share":>9s} {"GN GB/s":>8s}')
for B in a.batches:
    x = (torch.randn(B, 2, int(a.seconds * sr), generator=torch.Generator().manual_seed(B)) * 0.1).cuda()
    t_ours = timed(run_ours, x)
    t_hf = float('nan') if a.no_transformers else timed(run_hf, x)
    if not a.no_transformers:   # the decoders on the same codes (white-noise input leaves RVQ near-ties a code flip would amplify)
        codes, scales, pad = m.model.encode(x, None, a.bandwidth)
        got = m.model.decode(codes, scales, None, pad)[0]
        with torch.no_grad():
            ref = hf.decode(codes, scales, None, False, pad)[0]
        err = ((got - ref).abs().max() / ref.abs().max().clamp_min(1)).item()
    else:
        err = float('nan')
    gn_bytes.clear()
    m._gn_stats, m._gn_apply = stats_logged, apply_logged
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_ours(x)
        torch.cuda.synchronize()
    m._gn_stats, m._gn_apply = _stats, _apply
    tot = gn = 0.0
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
        tot += us
        if 'groupnorm' in ev.key:
            gn += us
    audio = B * a.seconds
    print(f'{B:3d} {audio:8.0f} {t_ours:8.3f} {t_hf:8.3f} {t_hf / t_ours:8.2f} {audio / t_ours:15.1f} '
          f'{audio * sr / t_ours / 1e6:10.2f} {gn / tot:9.1%} {sum(gn_bytes) / (gn * 1e-6) / 1e9:8.0f}   (decoder max err vs hf on the same codes, relative to max(1, peak) {err:.1e})')
    if B == a.batches[-1]:
        print(prof.key_averages().table(sort_by='self_device_time_total' if hasattr(prof.key_averages()[0], 'self_device_time_total')
                                        else 'self_cuda_time_total', row_limit=14))
