"""Stereo MusicGen against mono (synthetic weights of the released architectures): `MusicGen.generate` wall time and audio-s/s
of stereo-medium (8 interleaved codebooks, stereo codec) and medium (4 codebooks, mono codec) on the same GPU, the LM
generation and the codec decode also timed on their own.  Each model is warmed up with one call of the same shape, then
timed over --reps calls alternating the two models; the best call counts.  Prints the card name and power limit beside the
numbers.
    python profiles/perf_stereo.py [--batch 8] [--seconds 30] [--reps 2] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200.loaders import load_musicgen  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=8)
ap.add_argument('--seconds', type=float, default=30.0)
ap.add_argument('--reps', type=int, default=2)
ap.add_argument('--out', default=None)
a = ap.parse_args()
assert torch.cuda.is_available(), "this measurement needs the GPU"

gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                     text=True).stdout.strip()
descs = [f'description {b}' for b in range(a.batch)]
models = {}
for label, name in (('stereo_medium', 'synthetic/stereo-medium'), ('medium', 'synthetic/medium')):
    mg = load_musicgen(name)
    mg.set_generation_params(duration=a.seconds)
    mg.generate(descs)   # warm-up: allocates the caches of this shape and captures the step graph
    models[label] = mg


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


best = {k: dict(generate_s=float('inf'), lm_s=float('inf'), decode_s=float('inf')) for k in models}
for _ in range(a.reps):
    for label, mg in models.items():
        dt, _ = timed(lambda: mg.generate(descs))
        attrs, _ = mg._prepare_tokens_and_attributes(descs, None)
        lm_dt, tok = timed(lambda: mg._generate_tokens(attrs, None))
        dec_dt, wav = timed(lambda: mg.generate_audio(tok))
        b = best[label]
        b['generate_s'], b['lm_s'], b['decode_s'] = min(b['generate_s'], dt), min(b['lm_s'], lm_dt), min(b['decode_s'], dec_dt)
        b['tokens_shape'], b['wav_shape'] = list(tok.shape), list(wav.shape)

res = dict(gpu=gpu, batch=a.batch, seconds=a.seconds, reps=a.reps)
for label, b in best.items():
    b['audio_s_per_s'] = a.batch * a.seconds / b['generate_s']
    b['launches_per_step'] = models[label].lm.launches_per_step
    res[label] = b
res['stereo_over_mono_time'] = best['stereo_medium']['generate_s'] / best['medium']['generate_s']
print(json.dumps(res))
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'perf_stereo.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
