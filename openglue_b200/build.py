"""Build libopenglue_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m openglue_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libopenglue_b200.so')
SOURCES = ['api.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '--use_fast_math=false', '-Xcompiler', '-fPIC', '-shared', '-Xptxas', '-v']


def _nvcc() -> str:
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found (set NVCC=/path/to/nvcc)')


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, '..', 'include', 'openglue_b200.h')]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    flags = [f for f in NVCC_FLAGS if f != '--use_fast_math=false']
    cmd = [_nvcc(), *flags, '-o', LIB, *[os.path.join(CSRC, s) for s in SOURCES], '-lcudart']
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError(f'nvcc failed ({res.returncode}): {" ".join(cmd)}')
    with open(os.path.join(HERE, 'build.log'), 'w') as f:
        f.write(' '.join(cmd) + '\n' + res.stdout + res.stderr)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
