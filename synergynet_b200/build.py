"""Build the sm_90a C-ABI library in-tree with nvcc (no torch cpp_extension, no JIT cache).

``python -m synergynet_b200.build`` or ``__graft_entry__.build()``.  The resulting
``synergynet_b200/libsynergy_b200.so`` is git-ignored but travels with the work tree.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, 'csrc')
LIB_NAME = 'libsynergy_b200.so'
LIB_PATH = os.path.join(PKG_DIR, LIB_NAME)

NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '--use_fast_math=false', '-Xcompiler', '-fPIC', '-shared', '-Xptxas', '-v']


def _nvcc() -> str:
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found; cannot build the sm_90a library')


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(PKG_DIR, '..', 'include', 'synergy_b200.h'))
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB_PATH
    flags = [f for f in NVCC_FLAGS if f != '--use_fast_math=false']
    cmd = [_nvcc(), *flags, '-o', LIB_PATH, *_sources()]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
    if proc.returncode != 0:
        raise RuntimeError('nvcc failed building ' + LIB_NAME)
    with open(os.path.join(PKG_DIR, 'build_ptxas.log'), 'w') as f:
        f.write(proc.stdout + proc.stderr)
    return LIB_PATH


if __name__ == '__main__':
    print(build_library(force='--force' in sys.argv, verbose=True))
