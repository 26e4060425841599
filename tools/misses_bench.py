"""Cost of misses=True: cost_het_cluster with and without the out-of-memory attempts on C3-mpl6 and C4-mpl4, and the
latency of closest_misses(100).

Each configuration runs in a child process of its own (one library per process), and the children alternate round by
round, so that clock drift hits every configuration alike.  ``--parent-tree`` adds the built metis_b200 package of an
earlier commit (without misses) as a third configuration.  The card's power limit and clocks are queried in the same
session and printed with the times (ms).

    python tools/misses_bench.py [--rounds 3] [--reps 5] [--parent-tree dir/holding/metis_b200]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
WORKLOADS_RUN = ['c3_homo64_mpl6', 'c4_het128']


def child(tree: str, misses: bool, reps: int) -> dict:
    sys.path.insert(0, tree or ROOT)                      # the package (and its library) of this build
    import itertools
    import tempfile
    import torch
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    from metis_b200.workloads import WORKLOADS, materialize, profile_file_order
    out = {}
    for name in WORKLOADS_RUN:
        w = WORKLOADS[name]
        root = tempfile.mkdtemp(prefix='misses_bench_')
        materialize(w, root)
        cluster = GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
        profile, _ = ProfileDataLoader(os.path.join(root, 'profile'), profile_file_order(w)).load_profile_data_all()
        cfg = ModelConfig(model_name='t', num_layers=w.num_layers, sequence_length=w.sequence_length,
                          vocab_size=w.vocab_size, hidden_size=w.hidden_size, attention_head_size=32)
        args = parse_args(w.cli_args(root))
        seqs = list(itertools.permutations(w.device_types()))
        volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
        est = api.HeteroCostEstimator(profile, cfg, volume, cluster)
        bal = api.LayerLoadBalancer(cluster, profile, cfg, args.gbs)
        flags = dict(misses=True) if misses else {}
        api.cost_het_cluster(args, cluster, profile, cfg, est, bal, node_sequences=seqs, device='cuda:0', **flags)
        search_s, total_s, res = [], [], None
        for _ in range(reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            res = api.cost_het_cluster(args, cluster, profile, cfg, est, bal, node_sequences=seqs, device='cuda:0',
                                       **flags)
            total_s.append(time.perf_counter() - t)
            search_s.append(res.timings['gpu_search_s'])
        row = dict(search_ms=1e3 * statistics.median(search_s), total_ms=1e3 * statistics.median(total_s),
                   candidates=len(res))
        if misses:
            row['misses'] = len(res.misses)
            row['misses_ms'] = 1e3 * res.timings['misses_s']
            lat = []
            for _ in range(3):
                res._closest = None
                t = time.perf_counter()
                res.closest_misses(100)
                lat.append(time.perf_counter() - t)
            row['closest_100_ms'] = 1e3 * min(lat)
        out[name] = row
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--parent-tree', default='')
    ap.add_argument('--child', default='')
    a = ap.parse_args()
    if a.child:
        tree, misses = a.child.rsplit(':', 1)
        print(json.dumps(child(tree, misses == '1', a.reps)))
        return
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    configs = [('plain', ':0'), ('misses', ':1')] + ([('parent', f'{a.parent_tree}:0')] if a.parent_tree else [])
    runs = {k: [] for k, _ in configs}
    for _ in range(a.rounds):
        for key, spec in configs:
            p = subprocess.run([sys.executable, __file__, '--child', spec, '--reps', str(a.reps)], capture_output=True,
                               text=True, cwd=ROOT)
            if p.returncode:
                raise SystemExit(p.stderr)
            runs[key].append(json.loads(p.stdout.strip().splitlines()[-1]))
    print(json.dumps(dict(gpu=smi, runs=runs), indent=1))


if __name__ == '__main__':
    main()
