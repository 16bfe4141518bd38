"""Paged KV cache for continuous batching (`continuous(kv_cache_gb=...)`), on synthetic MusicGen-medium and -large.

1. The decode step, paged against contiguous, at equal slots and at KV lengths of about 1 and about 1500 positions: CUDA
   events over the captured step graph, the two layouts alternated `--reps` times in this one command (the spread of the
   repeats is printed beside the means).  Every slot decodes; the long case starts each slot at column 1400.
2. MusicGen-medium, the workload of profiles/perf_continuous.py (text requests of {5, 10, 20, 30} s, `--requests` of them):
   contiguous 64 slots against paged sessions at 96 and 128 slots whose pool is what the contiguous 64 slots reserve.
   Reports audio-s/s (codec decode included, each run ending in a device synchronise), occupancy, peak and mean pages in
   use, and the time the head request waited for pages with a slot free (wall time of the polls in which it waited).
3. MusicGen-large: the largest contiguous session that fits, against paged sessions at 64 and 96 slots with its reservation.
Every shape is warmed up first.  Prints the card name and power limit beside the numbers.
    python profiles/perf_continuous_paged.py [--parts step medium large] [--requests 128 256] [--reps 3] [--out DIR]"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

# sessions of 20-60 GB are built and freed one after another: without expandable segments the caching allocator's freed
# blocks fragment and a later pool of the same size does not fit
os.environ.setdefault('PYTORCH_CUDA_ALLOC_CONF', 'expandable_segments:True')
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200 import _lib  # noqa: E402
from audiocraft_b200.batching import PagePool, Request, SlotSession, kv_page_bytes  # noqa: E402
from audiocraft_b200.loaders import load_musicgen  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--requests', type=int, nargs='+', default=[128, 256])
ap.add_argument('--reps', type=int, default=3)
ap.add_argument('--step-iters', type=int, default=50)
ap.add_argument('--seed', type=int, default=0)
ap.add_argument('--parts', nargs='+', default=['step', 'medium', 'large'], choices=['step', 'medium', 'large'])
ap.add_argument('--out', default=None)
a = ap.parse_args()
assert torch.cuda.is_available(), "this measurement needs the GPU"

gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                     text=True).stdout.strip()
res = dict(gpu=gpu, step=[], medium=[], large=[])
print(f'# {gpu}', flush=True)


def workload(n, seed):
    g = torch.Generator().manual_seed(seed)
    choices = [5.0, 10.0, 20.0, 30.0]
    durations = [choices[int(i)] for i in torch.randint(0, 4, (n,), generator=g)]
    return durations, [f'request {i}: a piece of music number {i}' for i in range(n)]


def release(mg):
    """Drop the LM's session and handle so the next session's cache can take the memory."""
    mg.lm._session = None
    mg.lm._destroy()
    mg.lm._shape = None
    gc.collect()
    torch.cuda.empty_cache()


def serve(mg, slots, durations, descs, kv_cache_gb=None):
    gen = mg.continuous(slots=slots, kv_cache_gb=kv_cache_gb)
    for d, t in zip(durations, descs):
        gen.submit(t, duration=d)
    sch, sess = gen.scheduler, gen.session
    wait_s, n = 0.0, 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    while gen.pending:
        w0, p0 = sch.page_wait_steps, time.perf_counter()
        n += len(gen.poll())
        if sch.page_wait_steps > w0:
            wait_s += time.perf_counter() - p0
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    assert n == len(durations)
    out = dict(slots=slots, wall_s=wall, audio_s_per_s=sum(durations) / wall, occupancy=sch.occupancy, steps=sch.steps_run)
    if sess.pages is not None:
        out.update(kv_cache_gb=kv_cache_gb, n_pages=sess.pages.n_pages, peak_pages=sess.pages.peak,
                   mean_pages=sch.page_steps / max(1, sch.steps_run), head_wait_steps=sch.page_wait_steps,
                   head_wait_s=wait_s)
    else:
        out.update(kv_cache_gb=2 * slots * (sess.max_prefix + sess.seq_len_max) * kv_page_bytes(mg.lm) / 64 / 1e9)
    del gen
    release(mg)
    return out


def step_ms(mg, slots, paged, start_col, iters):
    lm = mg.lm
    max_gen_len = int(mg.max_duration * mg.frame_rate)
    cond = lm._condition_tensors(mg._prepare_tokens_and_attributes(['x'], None)[0])[0]
    kv_pages = None
    if paged:
        S = max_gen_len + max(lm.pattern_provider.get_pattern(max_gen_len).delays) + 1
        kv_pages = slots * PagePool.need(S)
    sess = SlotSession(lm, slots, max_gen_len, kv_pages=kv_pages)
    for k in range(slots):
        sess.admit(k, Request(max_gen_len, cond, None, seed=k))
    if start_col:   # every slot at column start_col: its attention reads start_col + 1 positions (values are not checked)
        lm._bufs['slot_state'][:slots, 0] = start_col
    sess.steps(5)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    sess.steps(iters)
    e1.record()
    torch.cuda.synchronize()
    del sess
    release(mg)
    return e0.elapsed_time(e1) / iters


WARM = ([5.0] * 4, [f'warm-up {i}' for i in range(4)])   # every session shape and the codec, before the timed runs
mg = load_musicgen('synthetic/medium') if {'step', 'medium'} & set(a.parts) else None
# ---- 1. step time, alternating layouts
for slots in ((32, 64) if 'step' in a.parts else ()):
    for col in (0, 1400):
        step_ms(mg, slots, False, col, 5)
        step_ms(mg, slots, True, col, 5)          # warm both shapes
        c, p = [], []
        for _ in range(a.reps):
            c.append(step_ms(mg, slots, False, col, a.step_iters))
            p.append(step_ms(mg, slots, True, col, a.step_iters))
        row = dict(model='medium', slots=slots, kv_len=col + 1, contiguous_ms=c, paged_ms=p,
                   contiguous_mean=statistics.mean(c), paged_mean=statistics.mean(p),
                   ratio=statistics.mean(p) / statistics.mean(c))
        res['step'].append(row)
        print(json.dumps(row), flush=True)

# ---- 2. medium workload: contiguous 64 slots against paged 96 / 128 slots at its reservation
budget = None
for n in (a.requests if 'medium' in a.parts else ()):
    durations, descs = workload(n, a.seed)
    for slots, paged in ((64, False), (96, True), (128, True)):
        gb = budget if paged else None
        serve(mg, slots, *WARM, gb)
        r = serve(mg, slots, durations, descs, gb)
        if not paged:
            budget = r['kv_cache_gb']
        r.update(model='medium', requests=n, audio_s=sum(durations), mode='paged' if paged else 'contiguous')
        res['medium'].append(r)
        print(json.dumps(r), flush=True)
del mg
gc.collect()
torch.cuda.empty_cache()

# ---- 3. large: the largest contiguous session that fits, against paged 64 / 96 slots at its reservation
if 'large' in a.parts:
    mg = load_musicgen('synthetic/large')
    durations, descs = workload(a.requests[0], a.seed)
    r = None
    for slots in (64, 60, 56, 52, 48, 40, 32):   # the largest that runs the workload, codec decode included
        err = None
        try:
            serve(mg, slots, *WARM)
            r = serve(mg, slots, durations, descs)
        except (torch.OutOfMemoryError, RuntimeError) as e:
            err = f'{type(e).__name__}: {str(e)[:120]}'
        if r is not None:
            break
        release(mg)   # after the except block: its traceback holds the failed session's buffers
        print(f'# large contiguous {slots} slots: {err}', flush=True)
        res['large'].append(dict(model='large', slots=slots, mode='contiguous', error=err))
    r.update(model='large', requests=len(durations), audio_s=sum(durations), mode='contiguous (largest that fits)')
    res['large'].append(r)
    print(json.dumps(r), flush=True)
    for slots in (64, 96):
        rp = None
        try:
            serve(mg, slots, *WARM, r['kv_cache_gb'])
            rp = serve(mg, slots, durations, descs, r['kv_cache_gb'])
        except (torch.OutOfMemoryError, RuntimeError) as e:   # the pool fits, the rest of a wider session may not
            err = f'{type(e).__name__}: {str(e)[:160]}'
        if rp is None:
            release(mg)
            rp = dict(slots=slots, kv_cache_gb=r['kv_cache_gb'], error=err)
        rp.update(model='large', requests=len(durations), audio_s=sum(durations), mode='paged')
        res['large'].append(rp)
        print(json.dumps(rp), flush=True)

print(json.dumps(res))
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'perf_continuous_paged.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
