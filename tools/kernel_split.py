#!/usr/bin/env python3
"""Developer tool: per-kernel device time of one search, measured with torch.profiler (CUDA activities).

  python tools/kernel_split.py [--workload c3_homo64_mpl6] [--steps 20] [--warmup 3] [--json OUT]

The search is set up the way bench.py sets up its `value` region: host inputs materialised from the workload's
seeds, the problem and plan space resident on the device, every costed candidate's record written to HBM, and a
256 MiB write between steps to flush L2.  After the warm-up, `--steps` searches run under the profiler; each
kernel's device time is summed over the trace and divided by the step count.  Profile in a run of its own: the
trace slows the host, so take step times from bench.py.  Prints the card name and power limit beside the numbers.
"""
from __future__ import annotations

import argparse
import itertools
import json
import os
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, limit = [v.strip() for v in out[0].split(',')]
        return name, limit
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c3_homo64_mpl6')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--json', default=None, help='also write the result to this file')
    ns = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from metis_b200 import api, native, search
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    from metis_b200.workloads import WORKLOADS, materialize, profile_file_order

    if not torch.cuda.is_available():
        raise SystemExit('kernel_split.py needs a CUDA device')
    native.load_library()
    dev = torch.device('cuda:0')
    w = WORKLOADS[ns.workload]
    with tempfile.TemporaryDirectory() as tmp:
        materialize(w, tmp)
        args = parse_args(w.cli_args(tmp))
        cluster = GPUCluster(args.hostfile_path, args.clusterfile_path)
        profile_data, _ = ProfileDataLoader(args.profile_data_path, profile_file_order(w)).load_profile_data_all()
    cfg = ModelConfig(model_name=args.model_name, num_layers=args.num_layers, sequence_length=args.sequence_length,
                      vocab_size=args.vocab_size, hidden_size=args.hidden_size,
                      attention_head_size=args.attention_head_size)
    balancer = api.LayerLoadBalancer(cluster, profile_data, cfg, args.gbs)
    seqs = list(itertools.permutations(w.device_types()))
    problem, space, _ = api.het_problem(args, cluster, profile_data, cfg, balancer, seqs, device_rows=True)
    dp = search.DeviceProblem(problem, space, dev)
    probe = search.HetSearcher(dp, 0, 1, 128, want_records=True, want_detail=False)
    stream = torch.cuda.current_stream(dev)
    ref = probe.run(stream)
    full = search.HetSearcher(dp, 0, 1, 128, want_records=True, want_detail=False, capacity=len(ref.records) + 1024)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    for _ in range(max(ns.warmup, 1)):
        full.launch(stream)
    stream.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(ns.steps):
            flush.fill_(i & 0xFF)
            full.launch(stream)
        stream.synchronize()

    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name
        if name.startswith('void '):
            name = name[5:]
        name = name.split('(')[0]
        t = e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total
        k = per.setdefault(name, [0.0, 0])
        k[0] += t
        k[1] += 1
    # the L2 flush is the one uint8 fill kernel per step (flush.fill_ above); everything else belongs to the search
    flush = [n for n in per if 'FillFunctor<unsigned char>' in n]
    if len(flush) != 1 or per[flush[0]][1] != ns.steps:
        raise SystemExit(f'cannot tell the L2 flush from the search kernels: {sorted(per)}')
    flush_us = per[flush[0]][0]
    search_us = sum(v[0] for v in per.values()) - flush_us
    rows = sorted(((v[0] / ns.steps / 1e3, v[1] // ns.steps, n) for n, v in per.items()), reverse=True)
    name, limit = card()
    print(f'{ns.workload}: {space.num_plans} plans, {ns.steps} searches under torch.profiler on {name}, '
          f'power limit {limit}')
    print(f'  search kernels {search_us / ns.steps / 1e3:.3f} ms per search (L2 flush excluded)')
    for ms, calls, n in rows:
        share = 100.0 * ms * 1e3 * ns.steps / search_us if search_us else 0.0
        flag = '  (L2 flush)' if n == flush[0] else ''
        print(f'  {ms:8.3f} ms  {share:5.1f} %  x{calls:<3d} {n}{flag}')
    if ns.json:
        with open(ns.json, 'w') as f:
            json.dump({'workload': ns.workload, 'gpu': name, 'power_limit': limit, 'steps': ns.steps,
                       'search_ms': search_us / ns.steps / 1e3,
                       'kernels': [{'name': n, 'ms': ms, 'calls': c} for ms, c, n in rows]}, f, indent=1)


if __name__ == '__main__':
    main()
