#!/usr/bin/env python3
"""Developer tool: run one search with the phase-clock build of the library and print where the chain kernel's
warp-cycles go.

  python tools/phase_profile.py [workload] [--build]

The phase-clock build is libmetis_b200_prof.so next to libmetis_b200.so: the same sources compiled with
-DMETIS_PROFILE_PHASES (metis_b200.build.build_library(profile=True); --build makes it first).  Its chain kernel
reads clock64() on the leader lane of every warp at each phase mark (metis_coop.cuh, WarpCoop::mark) and at each
block gate (ChainCoop::gate).  Printed per phase: share of the chain warps' cycles and cycles per balancer run of
the chain kernel (total cycles of the phase over the runs; the time a warp spends waiting in a gate is the phase
`gate wait`), and the histogram of the gate spread: per block and gate, the cycles from the first working warp's
arrival to the last one's, i.e. how long the fastest warp waits for the slowest.

--bulk prints the bulk round (het_first_kernel) instead: its phase clock runs on the lowest lane of each warp's
current group from one hook (DeviceSink::phase, Lockstep::mark) to the next.  Printed per phase: share of the bulk
round's warp-cycles, cycles per batch of 32 plans (one warp in lockstep) and per plan (a batch's cycles / 32)."""
import argparse
import ctypes
import itertools
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from metis_b200 import build, flatten, native, search  # noqa: E402
from metis_b200.data_loader import ProfileDataLoader  # noqa: E402
from metis_b200.gpu_cluster import GPUCluster  # noqa: E402
from metis_b200.utils import ModelConfig  # noqa: E402
from metis_b200.workloads import WORKLOADS, materialize, profile_file_order  # noqa: E402

NAMES = {0: 'fetch+decode', 1: 'begin+strategy', 2: 'P perf', 9: 'R init', 10: 'R fwd walk', 19: 'R fwd replay',
         18: 'R seq forward',
         11: 'R backward', 12: 'R leftovers', 17: 'R middle', 13: 'R vote', 14: 'R cnt+capa', 15: 'R adjust',
         16: 'R part', 20: 'M demand', 21: 'M reweight', 22: 'C stage terms', 23: 'C sums+emit', 24: 'chain advance',
         25: 'drain', 30: 'gate wait'}
RUNS, GATES, SPREAD, WARPS, HIST = 32, 33, 34, 35, 40     # WarpCoop's kMark* slots
BULK_NAMES = {1: 'P performance', 2: 'R init', 10: 'R forward', 11: 'R backward', 12: 'R leftovers', 13: 'R vote',
              14: 'R capacities', 15: 'R adjust', 16: 'R part', 3: 'M memory', 21: 'M reweight', 4: 'C cost'}
BULK_BATCHES = 31                                         # kBulkBatches (metis_eval.cuh)


def print_bulk(name, ms, marks):
    batches = marks[BULK_BATCHES] or 1
    tot = sum(marks[i] for i in BULK_NAMES) or 1
    print(f'{name}: {ms:.2f} ms (phase-clock build), bulk round: {marks[BULK_BATCHES]} batches of 32 plans, '
          f'{tot / 1e6:.1f} M warp-cycles, {tot / batches:.0f} per batch')
    print(f'  {"phase":<16s} {"share":>7s} {"cycles/batch":>13s} {"cycles/plan":>12s}')
    for i in BULK_NAMES:
        print(f'  {BULK_NAMES[i]:<16s} {100.0 * marks[i] / tot:6.1f}% {marks[i] / batches:13.0f} '
              f'{marks[i] / batches / 32:12.1f}')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('workload', nargs='?', default='c3_homo64_mpl6')
    ap.add_argument('--build', action='store_true', help='build libmetis_b200_prof.so first')
    ap.add_argument('--bulk', action='store_true', help='the bulk round (het_first_kernel) instead of the chain kernel')
    ns = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('phase_profile.py needs a CUDA device')
    prof = build.build_library(profile=True) if ns.build else build.PROF_LIB
    native._lib = native.load_library(prof)
    native._lib.metis_debug_marks.argtypes = [ctypes.c_void_p, ctypes.c_int]
    native._lib.metis_debug_bulk_marks.argtypes = [ctypes.c_void_p, ctypes.c_int]
    w = WORKLOADS[ns.workload]
    tmp = tempfile.mkdtemp()
    materialize(w, tmp)
    cluster = GPUCluster(tmp + '/hostfile', tmp + '/clusterfile.json')
    profile, _ = ProfileDataLoader(tmp + '/profile', profile_file_order(w)).load_profile_data_all()
    cfg = ModelConfig('SYN', w.num_layers, w.sequence_length, w.vocab_size, w.hidden_size, 32)
    seqs = list(itertools.permutations(w.device_types()))
    problem = flatten.build_problem(profile, cluster, cfg, w.gbs, w.max_tp, w.max_bs, seqs)
    space = flatten.build_plan_space(len(seqs), cluster.get_total_num_devices(), w.gbs, w.num_layers, w.variance,
                                     w.max_permute_len, native._lib)
    dp = search.DeviceProblem(problem, space, 'cuda:0')
    dp.lib = native._lib
    s = search.HetSearcher(dp, want_records=False)
    s.shard.reserved = int(os.environ.get('METIS_BULK_MIN', '0'))
    for _ in range(3):
        s.launch()
    torch.cuda.synchronize()
    marks = (ctypes.c_longlong * 64)()
    native._lib.metis_debug_marks(None, 1)
    native._lib.metis_debug_bulk_marks(None, 1)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); s.launch(); b.record(); torch.cuda.synchronize()
    sm = s.summary()
    if ns.bulk:
        bulk = (ctypes.c_longlong * 32)()
        native._lib.metis_debug_bulk_marks(ctypes.addressof(bulk), 0)
        print_bulk(ns.workload, a.elapsed_time(b), bulk)
        return
    native._lib.metis_debug_marks(ctypes.addressof(marks), 0)
    mt = sum(marks[:32]) or 1
    runs = marks[RUNS] or 1
    print(f'{ns.workload}: {a.elapsed_time(b):.2f} ms (phase-clock build), plans {space.num_plans}, admitted '
          f'{sm.reserved[0]}, chained {sm.reserved[1]}, B {sm.num_partition_calls}, runs {sm.num_balancer_runs} '
          f'(chain kernel {marks[RUNS]}), C {sm.num_records}')
    print(f'  chain kernel: {mt / 1e6:.1f} M leader-lane cycles over all warps, {mt / runs:.0f} per chain run')
    print(f'  {"phase":<16s} {"share":>7s} {"cycles/run":>11s}')
    for i in sorted(range(32), key=lambda i: -marks[i]):
        if marks[i]:
            print(f'  {NAMES.get(i, str(i)):<16s} {100.0 * marks[i] / mt:6.1f}% {marks[i] / runs:11.0f}')
    g = marks[GATES] or 1
    print(f'  gate spread (first to last working warp of a block): {marks[GATES]} gates, mean '
          f'{marks[SPREAD] / g:.0f} cycles, {marks[WARPS] / g:.1f} working warps per gate')
    for k in range(24):
        n = marks[HIST + k]
        if n:
            lo = 0 if k == 0 else 1 << k
            print(f'    [{lo:>8d}, {1 << (k + 1):>8d}) cycles  {n:8d}  {100.0 * n / g:5.1f}%')


if __name__ == '__main__':
    main()
