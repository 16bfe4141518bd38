"""Continuous batching of MusicGen-melody (synthetic weights of the medium architecture): 128 requests with seeded durations
drawn from {5, 10, 20, 30} s (the workload of perf_continuous.py), each with a seeded 30 s melody, a quarter of them null,
served by `MusicGen.continuous` at 32 (and 64) slots against `generate_with_chroma` in groups of 32 in arrival order and in
groups sorted by duration.  Reports audio-s/s (requested audio over wall time, codec decode included, each run ending in a
device synchronise) and the mean slot occupancy; the admission cost: one admission's prefix prefill (CUDA events,
acb_lm_admit_prefix minus the same admission without a prefix), its number of passes, and the share of each session's wall
time spent in admissions (CUDA events around every admission); and, as a check that the per-slot prefix costs a text model
nothing, the decode step of a full text-model session (synthetic MusicGen-medium) against `generate`'s at rows 64 and 128.
Every shape is warmed up first.  A 64-slot melody session needs about 68 GB of KV cache; when it does not fit it is
reported as not measured.  Prints the card name and power limit beside the numbers.
    python profiles/perf_continuous_melody.py [--requests 128] [--slots 32 64] [--group 32] [--seed 0] [--out DIR]"""
import argparse
import ctypes as C
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
mg = load_musicgen('synthetic/melody')
g = torch.Generator().manual_seed(a.seed)
choices = [5.0, 10.0, 20.0, 30.0]
durations = [choices[int(i)] for i in torch.randint(0, 4, (a.requests,), generator=g)]
descs = [f'request {i}: a piece of music number {i}' for i in range(a.requests)]
t30 = torch.arange(32000 * 30) / 32000
melodies = []
for i in range(a.requests):
    if i % 4 == 3:
        melodies.append(None)   # a null melody
    else:
        f = 110.0 * 2 ** (float(torch.randint(0, 24, (1,), generator=g)) / 12)
        melodies.append((0.3 * torch.sin(2 * torch.pi * f * t30) + 0.02 * torch.randn(t30.shape, generator=g))[None])
audio_s = sum(durations)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def run_continuous(slots, idx):
    gen = mg.continuous(slots=slots)
    events = []
    admit = gen.session.admit

    def timed_admit(slot, req):   # CUDA events around every admission (host work and prefix prefill)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        admit(slot, req)
        e1.record()
        events.append((e0, e1))
    gen.session.admit = timed_admit
    for i in idx:
        gen.submit(descs[i], duration=durations[i], melody=melodies[i],
                   melody_sample_rate=None if melodies[i] is None else 32000)
    n = sum(1 for _ in gen.run())
    assert n == len(idx)
    torch.cuda.synchronize()
    return gen.occupancy, sum(e0.elapsed_time(e1) for e0, e1 in events) / 1e3, len(events)


def run_groups(order):
    for k in range(0, len(order), a.group):
        grp = order[k:k + a.group]
        mg.set_generation_params(duration=max(durations[i] for i in grp))
        mg.generate_with_chroma([descs[i] for i in grp], [melodies[i] for i in grp], 32000)


res = dict(gpu=gpu, model='synthetic/melody', requests=a.requests, audio_s=audio_s, null_melodies=melodies.count(None),
           durations={str(c): durations.count(c) for c in choices}, runs=[], admission={}, text_step=[])
warm = list(range(min(a.requests, 8)))
run_groups(warm)                               # warm-up: the codec and the group shapes
arrival = list(range(a.requests))
by_len = sorted(arrival, key=lambda i: durations[i])
for name, order in ((f'generate_with_chroma groups of {a.group}, arrival order', arrival),
                    (f'generate_with_chroma groups of {a.group}, sorted by duration', by_len)):
    t, _ = timed(lambda: run_groups(order))
    res['runs'].append(dict(mode=name, wall_s=t, audio_s_per_s=audio_s / t))
for slots in a.slots:   # the largest last: its KV cache may leave no room for the codec
    try:
        run_continuous(slots, warm)            # warm-up: the session shape
        t, (occ, t_admit, n_admit) = timed(lambda: run_continuous(slots, range(a.requests)))
        res['runs'].append(dict(mode=f'continuous slots={slots}', wall_s=t, audio_s_per_s=audio_s / t, occupancy=occ,
                                admissions=n_admit, admit_s=t_admit, admit_share=t_admit / t))
    except torch.cuda.OutOfMemoryError as e:
        res['runs'].append(dict(mode=f'continuous slots={slots}',
                                result='not measured: out of memory (' + str(e).splitlines()[0] + ')'))
        mg.lm._destroy()
        mg.lm._shape = None
        torch.cuda.empty_cache()

# one admission's prefix prefill: acb_lm_admit_prefix with the request's prefix minus the same admission without it
lm = mg.lm
attributes, _ = mg._prepare_melody([descs[0]], [melodies[0]], 32000)
_, prefix = lm._condition_tensors(attributes)
prefix = prefix.to('cuda', torch.float32).contiguous()
P = prefix.shape[1]
max_gen_len = int(mg.max_duration * mg.frame_rate)
sess = SlotSession(lm, a.slots[0], max_gen_len)
req = Request(max_gen_len, None, None, seed=0, prefix=prefix)
sess.admit(0, req)
S = req.meta['S']
samp = C.byref(_lib.LMSampling(1, 1.0, 250, 0.0, 3.0, 0, 0, 0.0))
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
ms = {}
for what, (ptr, n) in (('without_prefix', (None, 0)), ('with_prefix', (prefix.data_ptr(), P))):
    times = []
    for it in range(6):
        torch.cuda.synchronize()
        e0.record()
        _lib.check(lm._lib.acb_lm_admit_prefix(lm._handle, 1, None, 0, ptr, n, S, C.c_uint64(it), samp, _lib.stream()))
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    ms[what] = min(times[1:])
per = _lib.ACB_LM_PREFILL_ROWS // 2
res['admission'] = dict(prefix_len=P, passes=-(-P // per), admit_ms=ms['with_prefix'], admit_without_prefix_ms=ms['without_prefix'],
                        prefix_prefill_ms=ms['with_prefix'] - ms['without_prefix'])


# the text-model session step at rows 64 and 128 (the per-slot prefix word is read by its embed, QKV and attention kernels)
def step_ms(lm_, setup, iters):
    setup()
    _lib.check(lm_._lib.acb_lm_steps(lm_._handle, 5, _lib.stream()), 'lm_steps')   # warm
    e0.record()
    _lib.check(lm_._lib.acb_lm_steps(lm_._handle, iters, _lib.stream()), 'lm_steps')
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


del sess, req
lm._destroy()
torch.cuda.empty_cache()
text = load_musicgen('synthetic/medium')
tlm = text.lm
cond = tlm._condition_tensors(text._prepare_tokens_and_attributes(['x'], None)[0])[0]
for slots in (32, 64):
    def session():
        s = SlotSession(tlm, slots, max_gen_len)
        for k in range(slots):
            s.admit(k, Request(max_gen_len, cond, None, seed=k))

    def plain():
        tlm._generate_begin(None, text._prepare_tokens_and_attributes(['x'] * slots, None)[0], None, max_gen_len, True, 1.0,
                            250, 0.0, 3.0, None, False, None, None)
    ts, tg = step_ms(tlm, session, a.step_iters), step_ms(tlm, plain, a.step_iters)
    res['text_step'].append(dict(rows=2 * slots, slot_step_ms=ts, generate_step_ms=tg, ratio=ts / tg))
torch.cuda.synchronize()
print(json.dumps(res))
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'perf_continuous_melody.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
