"""MusicGen-melody (synthetic weights of the released architecture): CUDA-event time of the condition-prefix prefill
(acb_lm_begin_prefix minus acb_lm_begin on the same rows) and whole generate_with_chroma throughput with a melody and with a
null melody.  Prints the card name and power limit beside the numbers.
    python profiles/perf_melody.py [--batch 8] [--seconds 30] [--melody-seconds 30] [--out DIR]"""
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
from audiocraft_b200.loaders import load_musicgen  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=8)
ap.add_argument('--seconds', type=float, default=30.0)
ap.add_argument('--melody-seconds', type=float, default=30.0)
ap.add_argument('--out', default=None)
a = ap.parse_args()
assert torch.cuda.is_available(), "this measurement needs the GPU"

gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                     text=True).stdout.strip()
mg = load_musicgen('synthetic/melody')
mg.set_generation_params(duration=a.seconds)
lm, B = mg.lm, a.batch
g = torch.Generator().manual_seed(0)
t = torch.arange(int(32000 * a.melody_seconds)) / 32000
melody = torch.stack([0.3 * torch.sin(2 * torch.pi * (220 + 40 * b) * t) for b in range(B)])[:, None]
melody = melody + 0.02 * torch.randn(melody.shape, generator=g)
descs = [f'melody {b}' for b in range(B)]
attributes, _ = mg._prepare_tokens_and_attributes(descs, None, list(melody))
_, prefix = lm._condition_tensors(attributes)
P = prefix.shape[1]
S = int(a.seconds * mg.frame_rate) + max(lm.cfg_dict['delays']) + 1
lm._ensure(2 * B, P + S, 1, B)
samp = _lib.LMSampling(1, 1.0, 250, 0.0, 3.0, 1, 0)
prefix = prefix.to('cuda', torch.float32).contiguous()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
res = {}
for what in ('begin', 'begin_prefix'):
    times = []
    for it in range(4):
        torch.cuda.synchronize()
        e0.record()
        if what == 'begin':
            _lib.check(lm._lib.acb_lm_begin(lm._handle, None, B, 2 * B, 0, S, C.byref(samp), _lib.stream()))
        else:
            _lib.check(lm._lib.acb_lm_begin_prefix(lm._handle, None, _lib.ptr(prefix), P, B, 2 * B, 0, S, C.byref(samp),
                                                   _lib.stream()))
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    res[what + '_ms'] = min(times[1:])
res['prefix_prefill_ms'] = res['begin_prefix_ms'] - res['begin_ms']
res['prefix_len'] = P
res['prefill_passes'] = -(-P // (_lib.ACB_LM_PREFILL_ROWS // (2 * B)))

for label, mel in (('melody', list(melody)), ('null_melody', [None] * B)):
    mg.generate_with_chroma(descs, mel, 32000)   # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mg.generate_with_chroma(descs, mel, 32000)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    res[f'{label}_s'] = dt
    res[f'{label}_audio_s_per_s'] = B * a.seconds / dt
res.update(gpu=gpu, batch=B, seconds=a.seconds, melody_seconds=a.melody_seconds)
print(json.dumps(res))
if a.out:
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'perf_melody.json'), 'w') as fh:
        json.dump(res, fh, indent=1)
