"""In-tree build of libmetis_b200.so (nvcc, sm_90a only)."""
from __future__ import annotations

import os
import shutil
import subprocess
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libmetis_b200.so')
SOURCES = ['metis_search.cu', 'metis_rank.cu', 'metis_enum.cpp']
HEADERS = ['metis_eval.cuh', 'metis_coop.cuh', 'metis_warp.cuh', 'metis_trace.cuh', 'metis_rows.cuh', 'metis_internal.h', os.path.join('..', '..', 'include', 'metis_b200.h')]

NVCC_FLAGS = ['-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo',
              '-fmad=false',            # parity: no FMA contraction (CPython evaluates a*b+c in two roundings)
              '-diag-suppress', '128,20168',   # unreachable loop in one instantiation; '#pragma unroll 0' = compiler default
              '-Xcompiler', '-fPIC', '-shared']


def nvcc_path() -> str:
    for cand in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found: cannot build libmetis_b200.so')


def stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps: List[str] = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return LIB
    cmd = [nvcc_path()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + \
          ['-o', LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f'nvcc failed:\n{proc.stdout}\n{proc.stderr}')
    if verbose:
        print(proc.stderr)
    return LIB
