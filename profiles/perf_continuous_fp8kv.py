"""FP8 self-attention KV pool for paged continuous batching (`continuous(kv_cache_gb=..., kv_cache_dtype='fp8')`), on
synthetic MusicGen-medium and -large.

1. step: the decode step, fp16-paged against fp8-paged, at 32, 64 and 128 slots and KV lengths 1, 750 and 1401: CUDA events
   over the captured step graph, the two formats alternated `--reps` times in this one command.  Every slot decodes; the
   longer cases start each slot at column 749 / 1400.
2. medium: the workload of profiles/perf_continuous.py (text requests of {5, 10, 20, 30} s, `--requests` of them) in a
   56.7 GB pool: fp16 at 64 and 96 slots against fp8 at 64, 96 and 128.  Reports audio-s/s (codec decode included),
   occupancy, peak and mean pages in use, and the time the head request waited for pages with a slot free.
3. large: synthetic MusicGen-large at 64 and 96 slots, fp16 and fp8, in a 61.5 GB pool.
4. divergence: synthetic medium (random weights, so the figures say how far the format moves the logits of an untrained
   network, not of a released checkpoint), one continuation prompt of 1000 columns consumed one column per step in an fp16
   and an fp8 session; at each step the CFG-mixed logits of both: the maximum |delta log-softmax| over the fp16 session's
   top 250 tokens of each codebook, the mean KL(fp16 || fp8), and the top-1 agreement.
Every shape is warmed up first.  Prints the card name and power limit beside the numbers.
    python profiles/perf_continuous_fp8kv.py [--parts step medium large divergence] [--requests 128 256] [--reps 3]
                                             [--out DIR]"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

os.environ.setdefault('PYTORCH_CUDA_ALLOC_CONF', 'expandable_segments:True')
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200.batching import PagePool, Request, SlotSession, kv_page_bytes  # noqa: E402
from audiocraft_b200.loaders import load_musicgen  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--requests', type=int, nargs='+', default=[128, 256])
ap.add_argument('--reps', type=int, default=3)
ap.add_argument('--step-iters', type=int, default=50)
ap.add_argument('--seed', type=int, default=0)
ap.add_argument('--parts', nargs='+', default=['step', 'medium', 'large', 'divergence'],
                choices=['step', 'medium', 'large', 'divergence'])
ap.add_argument('--out', default=None)
a = ap.parse_args()
assert torch.cuda.is_available(), "this measurement needs the GPU"

gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                     text=True).stdout.strip()
res = dict(gpu=gpu, step=[], medium=[], large=[], divergence=[])
print(f'# {gpu}', flush=True)


def workload(n, seed):
    g = torch.Generator().manual_seed(seed)
    choices = [5.0, 10.0, 20.0, 30.0]
    durations = [choices[int(i)] for i in torch.randint(0, 4, (n,), generator=g)]
    return durations, [f'request {i}: a piece of music number {i}' for i in range(n)]


def release(mg):
    mg.lm._session = None
    mg.lm._destroy()
    mg.lm._shape = None
    gc.collect()
    torch.cuda.empty_cache()


def serve(mg, slots, durations, descs, kv_cache_gb, dtype):
    gen = mg.continuous(slots=slots, kv_cache_gb=kv_cache_gb, kv_cache_dtype=dtype)
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
    out = dict(slots=slots, kv_dtype=dtype, kv_cache_gb=kv_cache_gb, wall_s=wall, audio_s_per_s=sum(durations) / wall,
               occupancy=sch.occupancy, steps=sch.steps_run, n_pages=sess.pages.n_pages, peak_pages=sess.pages.peak,
               mean_pages=sch.page_steps / max(1, sch.steps_run), head_wait_steps=sch.page_wait_steps, head_wait_s=wait_s)
    del gen
    release(mg)
    return out


def step_ms(mg, slots, dtype, start_col, iters):
    lm = mg.lm
    max_gen_len = int(mg.max_duration * mg.frame_rate)
    cond = lm._condition_tensors(mg._prepare_tokens_and_attributes(['x'], None)[0])[0]
    S = max_gen_len + max(lm.pattern_provider.get_pattern(max_gen_len).delays) + 1
    sess = SlotSession(lm, slots, max_gen_len, kv_pages=slots * PagePool.need(S), kv_dtype=dtype)
    for k in range(slots):
        sess.admit(k, Request(max_gen_len, cond, None, seed=k))
    if start_col:   # every slot at column start_col: its attention reads start_col + 1 positions (values are not checked)
        lm._bufs['slot_state'][:slots, 0] = start_col
    # positions the moved slots read were never written: zero K / V (and scales) in both formats, so both steps run the
    # attention, sampler and the rest on the same finite values
    for t in (sess.k_pool, sess.v_pool) + ((sess.k_scale, sess.v_scale) if dtype == 'fp8' else ()):
        t.view(torch.uint8).zero_()
    sess.steps(5)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    sess.steps(iters)
    e1.record()
    torch.cuda.synchronize()
    del sess
    release(mg)
    return e0.elapsed_time(e1) / iters


WARM = ([5.0] * 4, [f'warm-up {i}' for i in range(4)])
mg = load_musicgen('synthetic/medium') if {'step', 'medium', 'divergence'} & set(a.parts) else None
# ---- 1. step time, alternating formats
for slots in ((32, 64, 128) if 'step' in a.parts else ()):
    for col in (0, 749, 1400):
        fmts = []
        for dtype in ('fp16', 'fp8'):   # a pool of every slot at full length: 128 fp16 slots do not fit in 80 GB
            try:
                step_ms(mg, slots, dtype, col, 5)
                fmts.append(dtype)
            except torch.OutOfMemoryError:
                release(mg)
        t = {dtype: [] for dtype in fmts}
        for _ in range(a.reps):
            for dtype in fmts:
                t[dtype].append(step_ms(mg, slots, dtype, col, a.step_iters))
        row = dict(model='medium', slots=slots, kv_len=col + 1, **{f'{k}_ms': v for k, v in t.items()},
                   **{f'{k}_mean': statistics.mean(v) for k, v in t.items()})
        if len(fmts) == 2:
            row['ratio'] = row['fp8_mean'] / row['fp16_mean']
        res['step'].append(row)
        print(json.dumps(row), flush=True)

# ---- 2. medium workload in 56.7 GB
for n in (a.requests if 'medium' in a.parts else ()):
    durations, descs = workload(n, a.seed)
    for slots, dtype in ((64, 'fp16'), (96, 'fp16'), (64, 'fp8'), (96, 'fp8'), (128, 'fp8')):
        serve(mg, slots, *WARM, 56.7, dtype)
        r = serve(mg, slots, durations, descs, 56.7, dtype)
        r.update(model='medium', requests=n, audio_s=sum(durations), page_bytes=kv_page_bytes(mg.lm, dtype))
        res['medium'].append(r)
        print(json.dumps(r), flush=True)

# ---- 4. divergence of the logits, one prompt consumed one column per step
if 'divergence' in a.parts:
    lm = mg.lm
    g = torch.Generator().manual_seed(a.seed)
    cols, gen_len = 1000, 1010
    prompt = torch.randint(0, lm.card, (1, lm.n_q, cols), generator=g)
    cond = lm._condition_tensors(mg._prepare_tokens_and_attributes(['a steady groove'], None)[0])[0]
    logits = {}
    for dtype in ('fp16', 'fp8'):
        S = gen_len + max(lm.pattern_provider.get_pattern(gen_len).delays) + 1
        sess = SlotSession(lm, 1, gen_len, kv_pages=PagePool.need(S), kv_dtype=dtype, use_sampling=False)
        sess.admit(0, Request(gen_len, cond, prompt, seed=1))
        logits[dtype] = torch.stack([sess.step_logits()[0].cpu() for _ in range(cols)])   # [cols, K, card]
        del sess
        release(mg)
    l16, l8 = torch.log_softmax(logits['fp16'].double(), -1), torch.log_softmax(logits['fp8'].double(), -1)
    top = l16.topk(250, -1).indices
    dmax = (l16.gather(-1, top) - l8.gather(-1, top)).abs().amax().item()
    kl = (l16.exp() * (l16 - l8)).sum(-1).mean().item()
    agree = (l16.argmax(-1) == l8.argmax(-1)).double().mean().item()
    row = dict(model='medium (synthetic weights)', prompt_columns=cols, max_abs_dlogsoftmax_top250=dmax, mean_kl=kl,
               top1_agreement=agree)
    res['divergence'].append(row)
    print(json.dumps(row), flush=True)
del mg
gc.collect()
torch.cuda.empty_cache()

# ---- 3. large at 64 and 96 slots in 61.5 GB
if 'large' in a.parts:
    mg = load_musicgen('synthetic/large')
    durations, descs = workload(a.requests[0], a.seed)
    for slots, dtype in ((64, 'fp16'), (96, 'fp16'), (64, 'fp8'), (96, 'fp8')):
        r = None
        try:
            serve(mg, slots, *WARM, 61.5, dtype)
            r = serve(mg, slots, durations, descs, 61.5, dtype)
        except (torch.OutOfMemoryError, RuntimeError) as e:
            err = f'{type(e).__name__}: {str(e)[:160]}'
        if r is None:
            release(mg)
            r = dict(slots=slots, kv_dtype=dtype, kv_cache_gb=61.5, error=err)
        r.update(model='large', requests=len(durations), audio_s=sum(durations))
        res['large'].append(r)
        print(json.dumps(r), flush=True)

print(json.dumps(res))
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'perf_continuous_fp8kv.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
