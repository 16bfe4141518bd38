"""Decode-step timing at pinned KV lengths (MusicGen-medium, batch 8, CFG rows 16): CUDA-event time of the captured
step graph, and -- when run under `ncu --metrics gpu__time_duration.sum` -- a per-kernel launch list of one step at
KV length 750.   python profiles/perf_lm_step.py [--scale medium] [--one 750]"""
import argparse
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200 import _lib  # noqa: E402
from audiocraft_b200.loaders import load_lm_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--scale', default='medium')
ap.add_argument('--batch', type=int, default=8)
ap.add_argument('--one', type=int, default=-1, help='run a single direct (non-graph) step at this KV length and exit')
ap.add_argument('--reps', type=int, default=1, help='with --one: repeat the step')
a = ap.parse_args()

lm = load_lm_model(f'synthetic/{a.scale}')
B, S = a.batch, 1504
cross = torch.randn(2 * B, 16, lm.dim, device='cuda') * 0.1
cross[B:] = 0
lm._ensure(2 * B, S, 16, B)
samp = _lib.LMSampling(1, 1.0, 250, 0.0, 3.0, 1, 0)
lm._bufs['seq_mask'].fill_(1)
_lib.check(lm._lib.acb_lm_begin(lm._handle, _lib.ptr(cross), B, 2 * B, 16, S, C.byref(samp), _lib.stream()))
pos = lm._bufs['pos']
kv_tok = 2 * lm.dim * 2 * lm.num_layers
if a.one >= 0:
    for _ in range(a.reps):
        pos[0] = a.one
        torch.cuda.synchronize()
        _lib.check(lm._lib.acb_lm_step_logits(lm._handle, None, _lib.stream()))
        torch.cuda.synchronize()
    sys.exit(0)
print(f'launches/step={lm._lib.acb_lm_launches_per_step(lm._handle)} '
      f'W_step={lm.weight_bytes_per_step / 1e9:.2f} GB')
for t in (0, 375, 750, 1125, 1499):
    reps = 20
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for it in range(2):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            pos[0] = t          # (tiny memset kernel in the timed loop; same for every t)
            _lib.check(lm._lib.acb_lm_steps(lm._handle, 1, _lib.stream()))
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    byt = lm.weight_bytes_per_step + 2 * B * (t + 1) * kv_tok
    # the same step as direct stream launches (no graph): what the graph saves in launch overhead
    for it in range(2):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            pos[0] = t
            _lib.check(lm._lib.acb_lm_step_logits(lm._handle, None, _lib.stream()))
        e1.record()
        torch.cuda.synchronize()
    ms_direct = e0.elapsed_time(e1) / reps
    print(f'kv_len={t + 1:5d}  graph {ms:7.3f} ms/step  direct {ms_direct:7.3f} ms/step  algorithmic {byt / 1e9:.2f} GB -> '
          f'{byt / ms / 1e6:7.1f} GB/s')
