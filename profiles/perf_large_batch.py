"""Large batches on one GPU: one wide LM call (65-256 rows, the wgmma GEMM) against the same items split into calls of 32
(the mma.sync GEMM), the GEMM-only pass bandwidth at rows 64 / 128 / 256, the decode step at pinned KV lengths at rows 128
(profiles/perf_lm_step.py --batch 64), and the EnCodec decode of the same batches on its own.

    python profiles/perf_large_batch.py [--reps 2] [--skip-step]

Synthetic weights of the released architectures, sampling with top_k 250, cfg 3, text length 16, LM only and synchronised
for the audio-s/s figures.  Workloads are alternated and repeated; each figure prints every repeat."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audiocraft_b200 import _lib  # noqa: E402
from audiocraft_b200.loaders import load_compression_model, load_lm_model  # noqa: E402

HBM_BPS = 3.35e12   # H100 SXM data-sheet HBM3 bandwidth


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def reset(lm):
    lm._destroy()
    lm._shape = None
    torch.cuda.empty_cache()


def cross_for(lm, B, gen):
    cross = torch.randn(2 * B, 16, lm.dim, device='cuda', generator=gen) * 0.1
    cross[B:] = 0
    return cross


def generate_s(lm, cross, B, T):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    lm.generate(None, [], num_samples=B, max_gen_len=T, use_sampling=True, top_k=250, cfg_coef=3.0, cross_attention_src=cross)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def lm_throughput(lm, scale, dur, B, splits, reps):
    """audio-s/s of B items: one call, and `splits` sequential calls of B / splits items (same conditions)."""
    T = int(dur * 50)
    gen = torch.Generator(device='cuda').manual_seed(0)
    cross = cross_for(lm, B, gen)
    chunk = B // splits
    parts = [torch.cat([cross[i * chunk:(i + 1) * chunk], cross[B + i * chunk:B + (i + 1) * chunk]]) for i in range(splits)]
    lm._ensure(2 * B, T + 4, 16, B)   # one allocation for both variants
    generate_s(lm, parts[0], chunk, 8)   # warm-up: graph capture and module load of both GEMMs
    generate_s(lm, cross, B, 8)
    res = {'one call': [], f'{splits} x {chunk}': []}
    for _ in range(reps):
        res['one call'].append(B * dur / generate_s(lm, cross, B, T))
        res[f'{splits} x {chunk}'].append(B * dur / sum(generate_s(lm, p, chunk, T) for p in parts))
    for k, v in res.items():
        print(f'  {scale} {dur:g} s, B={B} {k:>8}: ' + ' / '.join(f'{x:6.2f}' for x in v) + ' audio-s/s', flush=True)
    reset(lm)


def gemm_pass(lm, scale, rows_list, launches=20):
    samp = _lib.LMSampling(1, 1.0, 250, 0.0, 3.0, 1, 0)
    for rows in rows_list:
        B = rows // 2
        reset(lm)
        lm._ensure(rows, 64, 16, B)
        cross = cross_for(lm, B, torch.Generator(device='cuda').manual_seed(1))
        _lib.check(lm._lib.acb_lm_begin(lm._handle, _lib.ptr(cross), B, rows, 16, 64, C.byref(samp), _lib.stream()))
        n = C.c_int(0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for it in range(2):   # the first round warms up
            torch.cuda.synchronize()
            e0.record()
            for _ in range(launches):
                _lib.check(lm._lib.acb_lm_debug_gemms(lm._handle, _lib.stream(), C.byref(n)))
            e1.record()
            torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / launches
        w = lm.weight_bytes_per_step
        kind = 'lm_gemm_wide_kernel' if rows > 64 else 'lm_gemm_kernel'
        print(f'  {scale} rows={rows:3d} ({kind}, {n.value} launches): {ms:6.3f} ms per pass, weights {w / 1e9:.2f} GB -> '
              f'{w / ms / 1e6:7.1f} GB/s = {w / ms / 1e-3 / HBM_BPS:.1%} of 3.35 TB/s', flush=True)
    reset(lm)


def encodec_decode(batches, reps):
    cm = load_compression_model('synthetic/encodec_32k')
    for B, dur in batches:
        codes = torch.randint(0, 2048, (B, 4, int(dur * 50)), device='cuda', generator=torch.Generator(device='cuda').manual_seed(2))
        cm.decode(codes[:, :, :50])
        ts = []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            cm.decode(codes)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        print(f'  EnCodec-32k decode B={B:3d} x {dur:g} s: ' + ' / '.join(f'{t:6.3f}' for t in ts) + ' s  '
              f'({B * dur / min(ts):.1f} audio-s/s)')
        del codes
        torch.cuda.empty_cache()
    del cm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--skip-step', action='store_true', help='skip the pinned-KV step times (perf_lm_step.py --batch 64)')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'perf_large_batch.py measures on the GPU'
    print(f'GPU: {gpu_info()}')
    if not a.skip_step:
        print('decode step at pinned KV lengths, MusicGen-medium rows 128 (perf_lm_step.py --batch 64):', flush=True)
        subprocess.run([sys.executable, os.path.join(ROOT, 'profiles', 'perf_lm_step.py'), '--batch', '64'], check=True)
    for scale, runs in (('medium', ((30, 64, 2), (10, 128, 4))), ('small', ((10, 128, 4),))):
        lm = load_lm_model(f'synthetic/{scale}')
        print(f'{scale}: GEMM-only pass (acb_lm_debug_gemms, CUDA events over 20 launches):', flush=True)
        gemm_pass(lm, scale, [64, 128, 256])
        print(f'{scale}: LMModel.generate, LM only, synchronised; the split calls are B = 32 each (repeats in order):', flush=True)
        for dur, B, splits in runs:
            lm_throughput(lm, scale, dur, B, splits, a.reps)
        del lm
        torch.cuda.empty_cache()
    print('EnCodec-32k decode of the same batches:', flush=True)
    encodec_decode([(32, 30), (64, 30), (32, 10), (128, 10)], a.reps)


if __name__ == '__main__':
    main()
