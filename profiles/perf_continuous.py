"""Continuous batching on synthetic MusicGen-medium: 128 text requests with seeded durations drawn from {5, 10, 20, 30} s,
served by `MusicGen.continuous` at 32 and 64 slots, against `generate` in groups of 32 in arrival order and in groups
sorted by duration (a group runs to its longest member).  Reports audio-s/s (requested audio over wall time, codec decode
included, each run ending in a device synchronise), the mean slot occupancy, and the decode step of a full session against
`generate`'s at equal rows (CUDA events over the captured step graph).  Every shape is warmed up first.  Prints the card
name and power limit beside the numbers.
    python profiles/perf_continuous.py [--requests 128] [--slots 32 64] [--group 32] [--seed 0] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200 import _lib  # noqa: E402
from audiocraft_b200.batching import Request, SlotSession  # noqa: E402
from audiocraft_b200.loaders import load_musicgen  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--requests', type=int, default=128)
ap.add_argument('--slots', type=int, nargs='+', default=[32, 64])
ap.add_argument('--group', type=int, default=32)
ap.add_argument('--seed', type=int, default=0)
ap.add_argument('--step-iters', type=int, default=50)
ap.add_argument('--out', default=None)
a = ap.parse_args()
assert torch.cuda.is_available(), "this measurement needs the GPU"

gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                     text=True).stdout.strip()
mg = load_musicgen('synthetic/medium')
g = torch.Generator().manual_seed(a.seed)
choices = [5.0, 10.0, 20.0, 30.0]
durations = [choices[int(i)] for i in torch.randint(0, 4, (a.requests,), generator=g)]
descs = [f'request {i}: a piece of music number {i}' for i in range(a.requests)]
audio_s = sum(durations)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def run_continuous(slots, idx):
    gen = mg.continuous(slots=slots)
    for i in idx:
        gen.submit(descs[i], duration=durations[i])
    n = sum(1 for _ in gen.run())
    assert n == len(idx)
    return gen.occupancy


def run_groups(order):
    for k in range(0, len(order), a.group):
        grp = order[k:k + a.group]
        mg.set_generation_params(duration=max(durations[i] for i in grp))
        mg.generate([descs[i] for i in grp])


def step_ms(setup, iters):
    """Mean time of one captured decode step (CUDA events over `iters` graph launches) after `setup()` began a generation."""
    setup()
    lm = mg.lm
    _lib.check(lm._lib.acb_lm_steps(lm._handle, 5, _lib.stream()), 'lm_steps')   # warm
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(lm._lib.acb_lm_steps(lm._handle, iters, _lib.stream()), 'lm_steps')
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


res = dict(gpu=gpu, model='synthetic/medium', requests=a.requests, audio_s=audio_s,
           durations={str(c): durations.count(c) for c in choices}, runs=[], step=[])
warm = list(range(min(a.requests, 8)))
for slots in a.slots:                          # warm-up: every session shape and the codec
    run_continuous(slots, warm)
run_groups(warm)
for slots in a.slots:
    t, occ = timed(lambda: run_continuous(slots, range(a.requests)))
    res['runs'].append(dict(mode=f'continuous slots={slots}', wall_s=t, audio_s_per_s=audio_s / t, occupancy=occ))
arrival = list(range(a.requests))
by_len = sorted(arrival, key=lambda i: durations[i])
for name, order in ((f'generate groups of {a.group}, arrival order', arrival),
                    (f'generate groups of {a.group}, sorted by duration', by_len)):
    t, _ = timed(lambda: run_groups(order))
    res['runs'].append(dict(mode=name, wall_s=t, audio_s_per_s=audio_s / t))

# the decode step at equal rows: a session with every slot decoding vs generate's graph, both at KV length ~1
max_gen_len = int(mg.max_duration * mg.frame_rate)
for slots in a.slots:
    lm = mg.lm
    cond = lm._condition_tensors(mg._prepare_tokens_and_attributes(['x'], None)[0])[0]

    def session():
        s = SlotSession(lm, slots, max_gen_len)
        for k in range(slots):
            s.admit(k, Request(max_gen_len, cond, None, seed=k))

    def plain():
        mg.set_generation_params(duration=mg.max_duration)
        lm._generate_begin(None, mg._prepare_tokens_and_attributes(['x'] * slots, None)[0], None, max_gen_len, True, 1.0,
                           250, 0.0, 3.0, None, False, None, None)

    ts, tg = step_ms(session, a.step_iters), step_ms(plain, a.step_iters)
    res['step'].append(dict(rows=2 * slots, slot_step_ms=ts, generate_step_ms=tg, ratio=ts / tg))
torch.cuda.synchronize()
print(json.dumps(res))
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'perf_continuous.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
