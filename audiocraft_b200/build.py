"""Build libaudiocraft_b200.so in-tree with nvcc for the H100 (sm_90a; cross-compiles without a GPU).

    python -m audiocraft_b200.build [--force]

The .so, the objects, the stamp and build.log are build products (git-ignored).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libaudiocraft_b200.so')
STAMP = LIB + '.stamp'
SOURCES = ['api.cu', 'encodec.cu', 'lm.cu']
HEADERS = ['common.cuh', 'gridbar.cuh', 'wgmma.cuh', os.path.join('..', '..', 'include', 'audiocraft_b200.h')]
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
FLAGS = ['-O3', '-std=c++17', '-lineinfo'] + ARCH + ['-Xcompiler', '-fPIC',
         '-Xptxas', '-v']
OBJ_SUFFIX = '.o'
LOG = os.path.join(HERE, 'build.log')
if os.environ.get('ACB_BUILD_VARIANT'):   # experiment builds: extra -D flags (ACB_BUILD_DEFS) into libaudiocraft_b200_<variant>.so; run with ACB_LIB=<path>
    _v = os.environ['ACB_BUILD_VARIANT']
    FLAGS += os.environ.get('ACB_BUILD_DEFS', '').split()
    LIB = os.path.join(HERE, f'libaudiocraft_b200_{_v}.so')
    STAMP = LIB + '.stamp'
    OBJ_SUFFIX = f'.{_v}.o'
    LOG = os.path.join(HERE, f'build_{_v}.log')


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), 'rb') as fh:
            h.update(fh.read())
    h.update(' '.join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIB
    objs = []
    procs = []
    for f in SOURCES:
        obj = os.path.join(CSRC, f.replace('.cu', OBJ_SUFFIX))
        objs.append(obj)
        cmd = [NVCC] + FLAGS + ['-c', os.path.join(CSRC, f), '-o', obj]
        procs.append((f, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    logs = []
    for f, p in procs:
        out, _ = p.communicate()
        logs.append(f'== {f}\n{out}')
        if p.returncode != 0:
            raise RuntimeError(f'nvcc failed on {f}:\n{out}')
    cmd = [NVCC, '-shared', '-o', LIB] + objs + ARCH + ['-lcudart']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f'link failed:\n{r.stdout}')
    with open(STAMP, 'w') as fh:
        fh.write(dig)
    with open(LOG, 'w') as fh:
        fh.write('\n'.join(logs))
    if verbose:
        print('\n'.join(logs))
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
