"""In-tree build of libmetis_b200.so (nvcc, sm_90a only)."""
from __future__ import annotations

import os
import shutil
import subprocess
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libmetis_b200.so')
PROF_LIB = os.path.join(HERE, 'libmetis_b200_prof.so')
SOURCES = ['metis_search.cu', 'metis_rank.cu', 'metis_select.cu', 'metis_recost.cu', 'metis_profile.cu', 'metis_noise.cu', 'metis_query.cu', 'metis_listing.cu', 'metis_enum.cpp']
HEADERS = ['metis_eval.cuh', 'metis_blob.cuh', 'metis_recost.cuh', 'metis_query.cuh', 'metis_noise.cuh', 'metis_coop.cuh', 'metis_warp.cuh', 'metis_trace.cuh', 'metis_rows.cuh', 'metis_comps.cuh', 'metis_internal.h', os.path.join('..', '..', 'include', 'metis_b200.h')]

NVCC_FLAGS = ['-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo',
              '-fmad=false',            # parity: no FMA contraction (CPython evaluates a*b+c in two roundings)
              '-diag-suppress', '128,20168',   # unreachable loop in one instantiation; '#pragma unroll 0' = compiler default
              '-Xcompiler', '-fPIC', '-shared']


def nvcc_path() -> str:
    for cand in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found: cannot build libmetis_b200.so')


def stale(lib: str = LIB) -> bool:
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    deps: List[str] = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False, profile: bool = False) -> str:
    """profile=True builds PROF_LIB instead: the same library with the chain kernel's phase clock
    (-DMETIS_PROFILE_PHASES, read by tools/phase_profile.py).  Never loaded by a search."""
    lib = PROF_LIB if profile else LIB
    if not force and not stale(lib):
        return lib
    cmd = [nvcc_path()] + NVCC_FLAGS + (['-DMETIS_PROFILE_PHASES'] if profile else []) + \
          (['-Xptxas', '-v'] if verbose else []) + ['-o', lib] + [os.path.join(CSRC, s) for s in SOURCES]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f'nvcc failed:\n{proc.stdout}\n{proc.stderr}')
    if verbose:
        print(proc.stderr)
    return lib
