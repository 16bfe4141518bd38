"""Prefilled prompts and window extension in continuous batching (`continuous(prefill_prompts=True)`) on synthetic
MusicGen-medium.

* Admission time against the prompt's prefilled columns (0, 100, 500, 600), contiguous and paged at 32 slots: the
  acb_lm_admit_prompt call between two device synchronises, median of --reps admissions into a slot of a full session.
* A prompt workload: the 128 requests of perf_continuous.py (durations from {5, 10, 20, 30} s), half of them continuations
  of a 5-10 s prompt (duration raised to prompt + 5 s where needed), at 32 and 64 slots with prefill_prompts False and True:
  audio-s/s (requested audio over wall time, codec decode included) and the median and p90 time from submit to result of
  the prompted requests (all requests are submitted at once).
* A long-form workload: 96 requests of 5-30 s and 32 of 45-120 s in a session of 32 slots (prefill_prompts=True, window
  extension) against `generate` in groups of 32 in arrival order (a group runs to its longest member), or of 16 or 8 where
  a group's codec decode does not fit in memory (recorded as such).
Every shape is warmed up first.  Prints the card name and power limit beside the numbers.
    python profiles/perf_continuous_prefill.py [--requests 128] [--slots 32 64] [--long 32] [--reps 5] [--seed 0]
        [--sections admission prompt long] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200.batching import PagePool, Request, SlotSession  # noqa: E402
from audiocraft_b200.loaders import load_musicgen  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--requests', type=int, default=128)
ap.add_argument('--slots', type=int, nargs='+', default=[32, 64])
ap.add_argument('--long', type=int, default=32, help='requests of 45-120 s in the long-form workload')
ap.add_argument('--reps', type=int, default=5)
ap.add_argument('--seed', type=int, default=0)
ap.add_argument('--sections', nargs='+', default=['admission', 'prompt', 'long'], choices=['admission', 'prompt', 'long'])
ap.add_argument('--out', default=None)
a = ap.parse_args()
assert torch.cuda.is_available(), "this measurement needs the GPU"

gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                     text=True).stdout.strip()
mg = load_musicgen('synthetic/medium')
lm, fr, sr = mg.lm, mg.frame_rate, mg.sample_rate
g = torch.Generator().manual_seed(a.seed)
choices = [5.0, 10.0, 20.0, 30.0]
durations = [choices[int(i)] for i in torch.randint(0, 4, (a.requests,), generator=g)]
descs = [f'request {i}: a piece of music number {i}' for i in range(a.requests)]
prompts = {}
for i in range(0, a.requests, 2):   # every other request continues a 5-10 s prompt
    p_s = 5.0 + 5.0 * float(torch.rand(1, generator=g))
    prompts[i] = 0.1 * torch.randn(1, int(p_s * sr), generator=g)
    durations[i] = max(durations[i], round(p_s + 5.0, 2))
res = dict(gpu=gpu, model='synthetic/medium', requests=a.requests, admission=[], prompt_workload=[], long_form=[])


def dump():
    """Print (and write) what is measured so far: each section adds to `res`."""
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'perf_continuous_prefill.json'), 'w') as fh:
            json.dump(res, fh, indent=1)


def sync_time():
    torch.cuda.synchronize()
    return time.perf_counter()


# ----------------------------------------------------------------------------- admission time against prompt length
if 'admission' in a.sections:
    max_gen_len = int(mg.max_duration * fr)
    cross = lm._condition_tensors(mg._prepare_tokens_and_attributes(['x'], None)[0])[0]
    for paged in (False, True):
        S = max_gen_len + max(lm.pattern_provider.delays) + 1
        sess = SlotSession(lm, 32, max_gen_len, kv_pages=PagePool.need(S) * 34 if paged else None)
        for k in range(1, 32):
            sess.admit(k, Request(max_gen_len, cross, None, seed=k))
        for cols in (0, 100, 500, 600):
            prompt = torch.randint(0, lm.card, (1, lm.n_q, cols), generator=torch.Generator().manual_seed(cols)) if cols else None
            times = []
            for r in range(a.reps + 1):   # the first admission of each length warms up
                req = Request(max_gen_len, cross, prompt, seed=r, prefill_cols=cols)
                t0 = sync_time()
                sess.admit(0, req)
                times.append(sync_time() - t0)
                sess.retire(0)
            times = sorted(times[1:])
            res['admission'].append(dict(paged=paged, prefill_cols=cols, admit_ms=1e3 * times[len(times) // 2],
                                         passes=-(-cols // 32)))
        del sess   # its page pool: the next session needs the memory
        torch.cuda.empty_cache()
    dump()


# ----------------------------------------------------------------------------- prompt workload
def serve(slots, prefill, idx, durs, prompt_of):
    gen = mg.continuous(slots=slots, prefill_prompts=prefill)
    ids = {}
    t0 = sync_time()
    for i in idx:
        p = prompt_of.get(i)
        ids[gen.submit(descs[i % len(descs)], duration=durs[i], prompt=p, prompt_sample_rate=None if p is None else sr)] = i
    done = {}
    for rid, _ in gen.run():
        done[ids[rid]] = time.perf_counter() - t0
    torch.cuda.synchronize()
    return time.perf_counter() - t0, done, gen


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(q * len(xs)))]


if 'prompt' in a.sections:
    warm = list(range(min(a.requests, 8)))
    for slots in a.slots:
        for prefill in (False, True):
            serve(slots, prefill, warm, durations, prompts)
    audio_s = sum(durations)
    for slots in a.slots:
        for prefill in (False, True):
            wall, done, gen = serve(slots, prefill, range(a.requests), durations, prompts)
            lat = [done[i] for i in prompts]
            res['prompt_workload'].append(dict(slots=slots, prefill_prompts=prefill, wall_s=wall, audio_s_per_s=audio_s / wall,
                                               prompted_median_s=pct(lat, 0.5), prompted_p90_s=pct(lat, 0.9),
                                               occupancy=gen.occupancy))
            dump()

# ----------------------------------------------------------------------------- long-form workload
if 'long' in a.sections:
    n_short, g = a.requests - a.long, torch.Generator().manual_seed(a.seed + 1)
    long_durs = [choices[int(i)] for i in torch.randint(0, 4, (n_short,), generator=g)] + \
        [[45.0, 60.0, 90.0, 120.0][int(i)] for i in torch.randint(0, 4, (a.long,), generator=g)]
    order = torch.randperm(len(long_durs), generator=g).tolist()
    long_durs = [long_durs[i] for i in order]
    mg.set_generation_params(duration=40.0)   # warm-up of the windowed generate path
    mg.generate(descs[:2])
    serve(32, True, [k for k, d in enumerate(long_durs) if d > 30][:2] + [0], long_durs, {})
    wall, done, gen = serve(32, True, range(len(long_durs)), long_durs, {})
    res['long_form'].append(dict(mode='continuous slots=32 prefill_prompts', wall_s=wall, audio_s=sum(long_durs),
                                 audio_s_per_s=sum(long_durs) / wall, window_readmissions=gen.scheduler.readmitted,
                                 occupancy=gen.occupancy))
    dump()
    del gen
    # generate in groups, arrival order; a group of 32 at 120 s needs its codec decode of 32 x 120 s at once, which may not
    # fit: that is recorded, and the next smaller group size is timed
    for size in (32, 16, 8):
        try:
            torch.cuda.empty_cache()
            t0 = sync_time()
            for k in range(0, len(long_durs), size):
                grp = list(range(k, min(k + size, len(long_durs))))
                mg.set_generation_params(duration=max(long_durs[i] for i in grp))
                mg.generate([descs[i % len(descs)] for i in grp])
            wall = sync_time() - t0
        except torch.OutOfMemoryError:
            res['long_form'].append(dict(mode=f'generate groups of {size}, arrival order', result='out of memory'))
            dump()
            continue
        res['long_form'].append(dict(mode=f'generate groups of {size}, arrival order', wall_s=wall, audio_s=sum(long_durs),
                                     audio_s_per_s=sum(long_durs) / wall))
        dump()
        break
