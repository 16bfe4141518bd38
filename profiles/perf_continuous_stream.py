"""Streamed continuous batching on synthetic MusicGen-medium: the request mix of perf_continuous.py (128 text requests with
seeded durations from {5, 10, 20, 30} s, all submitted at once) through `MusicGen.continuous` at 32 and 64 slots, without
`chunk_duration` and with chunks of 0.5 / 1 / 2 s, alternated in one command (the non-streamed session runs before and after
the streamed ones).  Reports audio-s/s (requested audio over wall time, codec decode included, each run ending in a device
synchronise), the time from submit to a request's first audio piece and to its final piece (p50 / p95; the non-streamed
session's final is its waveform), codec calls per poll, and the decode step of a full session with every request on the
default top-k 250 against a mix where every fourth request samples top-p 0.9 (CUDA events over the captured step graph).
Every shape is warmed up first.  Prints the card name and power limit beside the numbers.
    python profiles/perf_continuous_stream.py [--requests 128] [--slots 32 64] [--chunks 0.5 1 2] [--seed 0] [--out DIR]"""
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
ap.add_argument('--chunks', type=float, nargs='+', default=[0.5, 1.0, 2.0])
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


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(q * (len(xs) - 1))))]


def run(slots, idx, chunk, durations=durations):
    """One session over the requests idx; returns wall time, per-request first / final times after submit, polls, codec calls."""
    gen = mg.continuous(slots=slots, chunk_duration=chunk)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ids = {gen.submit(descs[i], duration=durations[i]): i for i in idx}
    first, final, polls = {}, {}, 0
    while gen.pending:
        events = gen.poll()
        polls += 1
        torch.cuda.synchronize()   # a piece is only out once the device has written it
        now = time.perf_counter() - t0
        for ev in events:
            rid = ev[0]
            if chunk is None:
                first.setdefault(rid, now)
                final[rid] = now
            else:
                if ev[1].shape[-1]:
                    first.setdefault(rid, now)
                if ev[-1]:
                    final[rid] = now
    wall = time.perf_counter() - t0
    assert len(final) == len(ids)
    calls = gen.stream.codec_calls if gen.stream is not None else None
    return wall, list(first.values()), list(final.values()), polls, calls


def step_ms(slots, top_p_every, iters):
    """Mean time of one captured step of a full session (CUDA events over `iters` graph launches); every `top_p_every`-th
    slot samples top-p 0.9, the rest the session's top-k 250."""
    lm = mg.lm
    max_gen_len = int(mg.max_duration * mg.frame_rate)
    cond = lm._condition_tensors(mg._prepare_tokens_and_attributes(['x'], None)[0])[0]
    s = SlotSession(lm, slots, max_gen_len)
    for k in range(slots):
        opts = dict(top_p=0.9, top_k=0) if top_p_every and k % top_p_every == 0 else {}
        s.admit(k, Request(max_gen_len, cond, None, seed=k, **opts))
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
for slots in a.slots:                          # warm-up: every session shape and the codec, streamed and not
    for chunk in [None] + a.chunks:
        run(slots, warm, chunk, [choices[0]] * a.requests)
for slots in a.slots:
    for chunk in [None] + a.chunks + [None]:
        wall, first, final, polls, calls = run(slots, range(a.requests), chunk)
        res['runs'].append(dict(slots=slots, chunk_s=chunk, wall_s=wall, audio_s_per_s=audio_s / wall,
                                first_p50_s=pct(first, 0.5), first_p95_s=pct(first, 0.95),
                                final_p50_s=pct(final, 0.5), final_p95_s=pct(final, 0.95), polls=polls,
                                codec_calls_per_poll=None if calls is None else calls / polls))
        print(json.dumps(res['runs'][-1]), flush=True)
for slots in a.slots:
    uni, mix = step_ms(slots, 0, a.step_iters), step_ms(slots, 4, a.step_iters)
    uni2 = step_ms(slots, 0, a.step_iters)
    res['step'].append(dict(rows=2 * slots, uniform_ms=[uni, uni2], quarter_top_p_ms=mix, ratio=mix / min(uni, uni2)))
torch.cuda.synchronize()
print(json.dumps(res))
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'perf_continuous_stream.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
