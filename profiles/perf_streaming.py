"""Streaming generation on synthetic MusicGen-medium: the time to the first yielded piece of `generate_stream`, and its total wall
time against `generate` in the same run, for B items of --seconds of audio and each chunk duration.  Every shape is warmed up
once; then each repetition alternates `generate` and `generate_stream` at every chunk duration, each call ending in a device
synchronise, and the best repetition counts.  Prints the card name and power limit beside the numbers.
    python profiles/perf_streaming.py [--batches 1 8] [--seconds 30] [--chunks 0.5 1 2] [--reps 2] [--out DIR]"""
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
ap.add_argument('--batches', type=int, nargs='+', default=[1, 8])
ap.add_argument('--seconds', type=float, default=30.0)
ap.add_argument('--chunks', type=float, nargs='+', default=[0.5, 1.0, 2.0])
ap.add_argument('--reps', type=int, default=2)
ap.add_argument('--out', default=None)
a = ap.parse_args()
assert torch.cuda.is_available(), "this measurement needs the GPU"

gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                     text=True).stdout.strip()
mg = load_musicgen('synthetic/medium')
mg.set_generation_params(duration=a.seconds)


def run_generate(descs):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mg.generate(descs)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def run_stream(descs, chunk):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first = None
    for wav in mg.generate_stream(descs, chunk_duration=chunk):
        if first is None and wav.shape[-1]:
            torch.cuda.synchronize()
            first = time.perf_counter() - t0
    torch.cuda.synchronize()
    return first, time.perf_counter() - t0


res = dict(gpu=gpu, model='synthetic/medium', seconds=a.seconds, reps=a.reps, cases=[])
for B in a.batches:
    descs = [f'description {b}' for b in range(B)]
    run_generate(descs)                       # warm-up of every shape the timed calls use
    for c in a.chunks:
        run_stream(descs, c)
    best = dict(generate_s=float('inf'), stream={c: dict(first_s=float('inf'), total_s=float('inf')) for c in a.chunks})
    for _ in range(a.reps):
        best['generate_s'] = min(best['generate_s'], run_generate(descs))
        for c in a.chunks:
            first, total = run_stream(descs, c)
            s = best['stream'][c]
            s['first_s'], s['total_s'] = min(s['first_s'], first), min(s['total_s'], total)
    for c in a.chunks:
        s = best['stream'][c]
        res['cases'].append(dict(batch=B, chunk_s=c, first_piece_s=s['first_s'], stream_total_s=s['total_s'],
                                 generate_s=best['generate_s'], stream_over_generate=s['total_s'] / best['generate_s']))
print(json.dumps(res))
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'perf_streaming.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
