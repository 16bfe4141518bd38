"""FP8 LM weights against fp16 on the same seeded synthetic weights, alternating the two in one process:
  1. decode-step time (captured graph replay, CUDA events) at rows 2, 16, 64, 128, 256 and KV length 750, and the decode
     GEMMs alone (acb_lm_debug_gemms) with their weight bytes over time as a share of the 3.35 TB/s data-sheet HBM figure;
  2. MusicGen.generate, medium, batch 8, 30 s: audio seconds per second;
  3. quality on synthetic medium: 1000 teacher-forced steps, top-1 agreement and mean KL(fp16 || FP8) of the CFG logits
     (seeded random weights, not a released checkpoint);
  4. compute_predictions, medium, batch 8, T 1500.
Prints the card, its power limit and SM clock first.

    python profiles/perf_fp8_weights.py [--scales small medium large] [--parts step generate quality forward]
"""
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
from audiocraft_b200.loaders import load_lm_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--scales', nargs='+', default=['small', 'medium', 'large'])
ap.add_argument('--rows', type=int, nargs='+', default=[2, 16, 64, 128, 256])
ap.add_argument('--parts', nargs='+', default=['step', 'generate', 'quality', 'forward'])
ap.add_argument('--reps', type=int, default=30)
ap.add_argument('--out', default=None)
a = ap.parse_args()
HBM = 3.35e12
DT = ('fp16', 'fp8')
results = {}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip()
    print('GPU:', q, flush=True)
    return q


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def step_part(scale):
    lms = {dt: load_lm_model(f'synthetic/{scale}', weight_dtype=dt) for dt in DT}
    out = {}
    for rows in a.rows:
        B = rows // 2
        S, kv = 800, 750
        lm = lms['fp16']
        cache = 2 * lm.num_layers * rows * lm.num_heads * S * 64 * 2
        if cache > 0.9 * torch.cuda.mem_get_info()[0]:
            print(f'{scale} rows={rows:3d}: skipped, the KV cache ({cache / 2 ** 30:.1f} GiB) does not fit beside the weights of '
                  'both models', flush=True)
            continue
        per = {}
        for rnd in range(2):   # alternate the two dtypes, keep the second round
            for dt in DT:
                lm = lms[dt]
                cross = torch.randn(rows, 16, lm.dim, device='cuda') * 0.1
                lm._ensure(rows, S, 16, B)
                lm._bufs['seq_mask'].fill_(1)
                samp = _lib.LMSampling(1, 1.0, 250, 0.0, 3.0, 1, 0)
                _lib.check(lm._lib.acb_lm_begin(lm._handle, _lib.ptr(cross), B, rows, 16, S, C.byref(samp), _lib.stream()))
                pos = lm._bufs['pos']

                def step():
                    pos[0] = kv
                    _lib.check(lm._lib.acb_lm_steps(lm._handle, 1, _lib.stream()))
                nl = C.c_int(0)

                def gemms():
                    _lib.check(lm._lib.acb_lm_debug_gemms(lm._handle, _lib.stream(), C.byref(nl)))
                ms, gms = timed(step, a.reps), timed(gemms, a.reps)
                wb = lm.weight_bytes_per_step
                per[dt] = dict(step_ms=ms, gemm_ms=gms, weight_gb=wb / 1e9, gemm_hbm_share=wb / (gms * 1e-3) / HBM,
                               launches=lm._lib.acb_lm_launches_per_step(lm._handle))
                lm._destroy()   # the KV cache of 256 rows of large is 28 GB: one handle at a time
                lm._shape = None
                torch.cuda.empty_cache()
        out[rows] = per
        print(f'{scale} rows={rows:3d} kv={kv}: ' + '  '.join(
            f"{dt} step {per[dt]['step_ms']:.3f} ms gemms {per[dt]['gemm_ms']:.3f} ms "
            f"({per[dt]['weight_gb']:.2f} GB, {100 * per[dt]['gemm_hbm_share']:.0f}% of 3.35 TB/s)" for dt in DT) +
            f"  step speed-up {per['fp16']['step_ms'] / per['fp8']['step_ms']:.3f}x", flush=True)
    for lm in lms.values():
        lm._destroy()
    del lms
    torch.cuda.empty_cache()
    return out


def generate_part():
    from audiocraft_b200.musicgen import MusicGen
    out = {}
    mgs = {dt: MusicGen.get_pretrained('synthetic/medium', weight_dtype=dt) for dt in DT}
    for rnd in range(2):
        for dt in DT:
            mg = mgs[dt]
            mg.set_generation_params(duration=30, top_k=250)
            torch.manual_seed(0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            wav = mg.generate(['a rock song with drums'] * 8)
            torch.cuda.synchronize()
            dtm = time.perf_counter() - t0
            out[dt] = dict(seconds=dtm, audio_s_per_s=8 * 30 / dtm)
    for dt in DT:
        print(f"generate medium B=8 30 s {dt}: {out[dt]['seconds']:.2f} s, {out[dt]['audio_s_per_s']:.1f} audio-s/s", flush=True)
    del mgs, wav
    torch.cuda.empty_cache()
    return out


def quality_part():
    lms = {dt: load_lm_model('synthetic/medium', weight_dtype=dt) for dt in DT}
    B, n = 2, 1000
    g = torch.Generator().manual_seed(1)
    lm = lms['fp16']
    seq = torch.randint(0, lm.card, (B, lm.n_q, n + 1), generator=g)
    cross = torch.randn(2 * B, 12, lm.dim, generator=g) * 0.3
    cross[B:] = 0
    logits = {}
    for dt in DT:
        logits[dt] = lms[dt].teacher_forced_logits(seq, cross, 3.0, n_steps=n).float()
    p16 = torch.log_softmax(logits['fp16'], -1)
    p8 = torch.log_softmax(logits['fp8'], -1)
    kl = (p16.exp() * (p16 - p8)).sum(-1).mean().item()
    top1 = (logits['fp16'].argmax(-1) == logits['fp8'].argmax(-1)).float().mean().item()
    print(f'quality synthetic medium ({n} teacher-forced steps, B={B}, CFG 3): top-1 agreement {100 * top1:.2f}%, '
          f'mean KL(fp16||fp8) {kl:.3e} nats', flush=True)
    del lms
    torch.cuda.empty_cache()
    return dict(top1=top1, kl=kl)


def forward_part():
    lms = {dt: load_lm_model('synthetic/medium', weight_dtype=dt) for dt in DT}
    B, T = 8, 1500
    g = torch.Generator().manual_seed(2)
    codes = torch.randint(0, 2048, (B, 4, T), generator=g).cuda()
    cross = (torch.randn(B, 16, lms['fp16'].dim, generator=g) * 0.3).cuda()
    out = {}
    for rnd in range(2):
        for dt in DT:
            out[dt] = timed(lambda: lms[dt].compute_predictions(codes, cross_attention_src=cross), 3)
    for dt in DT:
        print(f'compute_predictions medium B={B} T={T} {dt}: {out[dt]:.1f} ms', flush=True)
    del lms
    torch.cuda.empty_cache()
    return out


results['gpu'] = card()
if 'step' in a.parts:
    results['step'] = {s: step_part(s) for s in a.scales}
if 'generate' in a.parts:
    results['generate'] = generate_part()
if 'quality' in a.parts:
    results['quality'] = quality_part()
if 'forward' in a.parts:
    results['forward'] = forward_part()
results['gpu_after'] = card()
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, 'w') as fh:
        json.dump(results, fh, indent=1, default=str)
