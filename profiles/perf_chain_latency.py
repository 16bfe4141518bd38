"""Floor of a decode step made of N dependent kernels: time per kernel of a CUDA graph holding a chain of EMPTY kernels
(griddepcontrol.launch_dependents + griddepcontrol.wait + one global read-modify-write), with and without programmatic
(PDL) edges, for grid / block / shared-memory footprints like the decode step's kernels.
    python profiles/perf_chain_latency.py"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from audiocraft_b200 import _lib  # noqa: E402

L = _lib.lib()
scratch = torch.zeros(4, dtype=torch.int32, device='cuda')
us = C.c_float(0)
print('n_kernels  ctas threads  smem_KB  pdl   us/kernel')
for ctas, threads, smem in ((16, 256, 0), (132, 128, 0), (264, 128, 52), (384, 128, 15), (384, 256, 0), (592, 128, 52)):
    for pdl in (0, 1):
        _lib.check(L.acb_debug_chain_latency(532, ctas, threads, smem * 1024, pdl, 20, C.byref(us), _lib.ptr(scratch)), 'probe')
        print(f'{532:9d} {ctas:5d} {threads:7d} {smem:8d} {pdl:4d} {us.value:10.3f}')
